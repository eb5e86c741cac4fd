"""How the search behaves on inputs with many near-ties: smooth (low-frequency) images, flat images with faint noise,
and the bench's uniform-noise pair.  Prints the time of one forward and whether the SR images are finite."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')):
    sys.path.insert(0, p)
import torch
import torch.nn.functional as F
import bench
from c2m_b200.pipeline import RestorationPipeline, synthetic_pair

dev = torch.device('cuda:0')
pipe = RestorationPipeline(dev).load_state_dicts(*bench.seeded_weights()).place()
g = torch.Generator().manual_seed(11)


def smooth(n, size, cells, noise):
    base = torch.rand(n, 3, cells, cells, generator=g)
    img = F.interpolate(base, size=(size, size), mode='bicubic', align_corners=False)
    return (img + noise * torch.randn(n, 3, size, size, generator=g)).clamp(0, 1)


def case(name, lq, ref):
    up = F.interpolate(lq, scale_factor=4, mode='bicubic', align_corners=False).clamp(0, 1)
    ref = F.pad(ref, (0, 640 - ref.shape[-1], 0, 640 - ref.shape[-2]))
    x = [t.to(dev) for t in (lq, up, ref)]
    pipe.forward(*x)
    torch.cuda.synchronize()
    print(f'== {name}', flush=True)
    t = time.perf_counter()
    for _ in range(3):
        sr = pipe.forward(*x)
    torch.cuda.synchronize()
    print(f'   forward {1e3 * (time.perf_counter() - t) / 3:.1f} ms  finite {bool(torch.isfinite(sr).all())}', flush=True)


lq, _, ref = synthetic_pair(1234, 4, 160, 500)
case('uniform noise (bench)', lq, ref[..., :500, :500])
case('smooth 10x10 cells + 2% noise', smooth(4, 160, 10, 0.02), smooth(4, 500, 12, 0.02))
case('smooth 4x4 cells + 0.5% noise', smooth(4, 160, 4, 0.005), smooth(4, 500, 4, 0.005))
case('flat grey + 0.2% noise', (0.5 + 0.002 * torch.randn(4, 3, 160, 160, generator=g)).clamp(0, 1),
     (0.5 + 0.002 * torch.randn(4, 3, 500, 500, generator=g)).clamp(0, 1))
case('Ref = upsampled LR (self-similar)', smooth(4, 160, 10, 0.02), None or F.interpolate(smooth(4, 160, 10, 0.02), size=(500, 500), mode='bicubic'))
