"""Per-shape bounds for the conv3x3 launches of one step, next to the measured times of
tools/conv_shapes.py (its log is the argument).  Bounds, all per launch:
  tensor : 3 x algorithmic flops (hi*hi + hi*lo + lo*hi) at the H100 SXM data-sheet dense fp16 rate
  smem   : operand-fetch model of the wgmma kernel (DESIGN.md K5): per 128-pixel tile, 64-wide Cout slice and K=16
           step the tensor cores read 8 KB (x_hi, [W_hi|W_lo]) + 6 KB (x_lo, W_hi) from shared memory at
           128 B/clk/SM -> 112 clk
  hbm    : 4 B per input / output / residual element at the H100 SXM data-sheet HBM3 bandwidth
Data-sheet rates are for a 700 W card; a power-limited card reaches less.
"""
import ast
import re
import sys

PEAK_TF, PEAK_GBS, SMS, CLK_GHZ, SMEM_CLK_PER_STEP = 989.0, 3350.0, 132, 1.98, 112.0

rows = []
for ln in open(sys.argv[1]):
    m = re.match(r"(\(.*?\))\s+n=\s*(\d+) ms=\s*([\d.]+) \(\s*([\d.]+) us each\)", ln)
    if not m:
        continue
    B, cin, cout, H, W, ps, f32, res = ast.literal_eval(m.group(1))
    n, us = int(m.group(2)), float(m.group(4))
    px = B * H * W
    flops = 2.0 * cin * cout * 9 * px
    tiles = B * ((H + 15) // 16) * ((W + 7) // 8)
    slices = (cout + 63) // 64
    ksteps = 9 * 2 * ((cin + 31) // 32)                     # K chunks of 32 channels, two K=16 MMAs per tap
    t_tensor = 3 * flops / (PEAK_TF * 1e12) * 1e6
    t_smem = tiles * slices * ksteps * SMEM_CLK_PER_STEP / (SMS * CLK_GHZ * 1e3)
    t_hbm = 4.0 * px * (cin + cout + (cout if res else 0)) / (PEAK_GBS * 1e9) * 1e6
    bound = max(t_tensor, t_smem, t_hbm)
    which = 'tensor' if bound == t_tensor else 'smem' if bound == t_smem else 'hbm'
    rows.append((n * us, n, f'{cin}->{cout} @{H}x{W}' + (' +res' if res else '') + (' ps2' if ps else '') + (' fp32out' if f32 else ''),
                 us, t_tensor, t_smem, t_hbm, which, bound / us))
tot = sum(r[0] for r in rows)
print(f'| shape (B=4) | launches | measured us | tensor-issue us | smem-fetch us | HBM us | binding | bound / measured | share of class |')
print('|---|---:|---:|---:|---:|---:|---|---:|---:|')
for r in sorted(rows, reverse=True):
    print(f'| {r[2]} | {r[1]} | {r[3]:.0f} | {r[4]:.0f} | {r[5]:.0f} | {r[6]:.0f} | {r[7]} | {r[8]:.2f} | {r[0] / tot * 100:.1f}% |')
wb = sum(r[0] * r[8] for r in rows) / tot
print(f'\nclass total {tot / 1e3:.2f} ms; time-weighted bound / measured = {wb:.2f}')
