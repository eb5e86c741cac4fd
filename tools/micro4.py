"""BASELINE config 4 rows only (quick check of the DCN microbenchmark)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'tools'), ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')]
import torch, microbench
dev = torch.device('cuda:0')
flush = torch.empty(192 << 20, dtype=torch.uint8, device=dev)
for r in microbench.run_config4(dev, flush, 3350.0):   # H100 SXM data-sheet HBM3 bandwidth, GB/s
    print(json.dumps(r))
