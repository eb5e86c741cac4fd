"""The three DCN layers of the BASELINE config-2 network (B=4 per GPU) in isolation: device time per launch (library
CUDA-event hook), algorithmic GB/s (SURVEY §8d bytes) and fraction of the measured HBM peak.  Random index map (what
the bench's random-weight features produce), octet-planar offsets, PSA in / out — exactly the fused path's call.
env LAYER in {small, medium, large, all}, B (4), N launches (5), COUT (default: C; e.g. COUT=64 times one 64-wide
output slice of a layer).  One process times every layer asked for; the first line names the card, its power limit
and SM clocks.  Also the target of the ncu capture of dcn_umma."""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200')]
import torch
from c2m_b200 import ops
dev = torch.device('cuda:0')
B, N, which = int(os.environ.get('B', '4')), int(os.environ.get('N', '5')), os.environ.get('LAYER', 'all')
cout_env = os.environ.get('COUT')
try:
    card = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit,clocks.sm,'
                           'clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
except OSError:
    card = f'{torch.cuda.get_device_name(dev)} (power limit and clocks not readable)'
print(f'card: {card}', flush=True)
pk = os.path.join(ROOT, 'MEASURED_PEAKS.json')
hbm = (json.load(open(pk)) if os.path.exists(pk) else {}).get('hbm_gbs', 6650.0)
flush = torch.empty(192 << 20, dtype=torch.uint8, device=dev)
g = torch.Generator().manual_seed(7)
for name, C, H, sc in (('small', 256, 160, 1), ('medium', 128, 320, 2), ('large', 64, 640, 4)):
    if which not in ('all', name):
        continue
    dg, gh = 8, 158
    x = torch.randn(B, C, H, H, generator=g).to(dev)
    cout = int(cout_env or C)
    w = (torch.randn(cout, C, 3, 3, generator=g) * 0.05).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    idx = torch.randint(0, gh * gh, (B, gh, gh), generator=g).to(dev)
    c8 = (27 * dg + 7) // 8
    om = torch.zeros(B, c8, H, H, 8, device=dev)
    om.view(B, c8, H * H, 8)[:, :18] = (torch.randn(B, 18, H * H, 8, generator=g) * 0.5).to(dev)
    om.view(B, c8, H * H, 8)[:, 18:] = torch.randn(B, 9, H * H, 8, generator=g).to(dev)
    om_oct = ops.OctF32(om, 27 * dg)
    xp = ops.psa_from_f32(x)
    del x
    ops.profile_enable(True)
    for i in range(N + 2):
        if i == 2:
            torch.cuda.synchronize(); ops.profile_collect('dcn')
        flush.fill_(1)
        ops.dcn_v2_fused_tc(xp, om_oct, w, b, dg, idx=idx, pre_scale=sc, lrelu=True, psa_out=True, out_f32=False)
    torch.cuda.synchronize()
    r = ops.profile_collect('dcn'); ops.profile_enable(False)
    ms = r['ms'] / r['launches']
    gbs = r['bytes'] / r['launches'] / ms / 1e6
    print(f'dcn {name}: C={C} Cout={cout} {H}x{H} B={B}: {ms:.3f} ms per launch, {gbs:.0f} GB/s algorithmic = {gbs / hbm:.3f} of measured HBM peak, '
          f'{r["flops"] / r["launches"] / ms / 1e9:.1f} TFLOP/s', flush=True)
