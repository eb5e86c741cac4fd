"""Time the tensor-core 3x3 convolution (PSA in and out, ReLU) on four layer shapes: CUDA events over 10 launches each."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200')]
import torch
from c2m_b200 import ops
dev = torch.device('cuda:0')
for (cin, cout, H) in ((64, 64, 640), (64, 64, 160), (128, 64, 640), (256, 256, 160)):
    x = torch.randn(4, cin, H, H, device=dev); w = torch.randn(cout, cin, 3, 3, device=dev) * 0.05; b = torch.randn(cout, device=dev)
    xp = ops.psa_from_f32(x); yp = ops.PSA.empty(4, cout, H, H, dev)
    for _ in range(3): ops.conv3x3_psa(xp, w, b, act='relu', out=yp)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): ops.conv3x3_psa(xp, w, b, act='relu', out=yp)
    e1.record(); torch.cuda.synchronize()
    print(f'{cin}->{cout}@{H}: {e0.elapsed_time(e1) / 10:.3f} ms', end='   ')
print()
