"""Small-shape pass over every kernel for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')):
    sys.path.insert(0, p)
import numpy as np
import torch
import seeding
import c2m_b200 as c2m
from c2m_b200 import ops
dev = 'cuda:0'
fin, fref = seeding.unit_features(1, 64, 24, 26).to(dev), seeding.unit_features(2, 64, 40, 22).to(dev)
for force in (False, True):
    idx, val = c2m.corr_argmax(fin[None], fref[None], norm_input=True, l2norm=True, force_generic=force)
pre = c2m.offset_pyramid(idx[:, :10, :10].contiguous() % 100, 2)
x = seeding.randn(3, (1, 64, 24, 24)).to(dev)
om = seeding.randn(4, (1, 216, 24, 24), 0.7).to(dev)
w = seeding.randn(5, (64, 64, 3, 3), 0.1).to(dev)
b = seeding.randn(6, (64,)).to(dev)
i2 = torch.randint(0, 100, (1, 10, 10), device=dev)
y1 = c2m.dcn_v2_fused_forward(x, om, w, b, 8, idx=i2, pre_scale=2, lrelu_slope=0.1)
yp, y2 = ops.dcn_v2_fused_tc(x, om, w, b, 8, idx=i2, pre_scale=2, lrelu=True, psa_out=True, out_f32=True)
xp = ops.psa_from_f32(x)
a = ops.conv3x3_psa(xp, w, b, act='relu')
c = ops.conv3x3_psa(a, w, b, residual=xp, residual2=a)
wbig = seeding.randn(7, (256, 128, 3, 3), 0.05).to(dev)
d = ops.conv3x3_psa(xp, wbig, None, x2=a, act='lrelu', pixel_shuffle=2)
e = ops.conv3x3_psa(xp, wbig[:216, :64].contiguous(), None, psa_out=False, out_f32=True)
# the literal `_ext` boundary on the tensor-core route, the max-pool, the PSA round trip and the tensor-core DCN on a PSA
# input (its operand from c2m_dcn_tc_operand_psa)
import _ext
off = seeding.randn(8, (1, 144, 24, 24), 2.0).to(dev)
msk = torch.sigmoid(seeding.randn(9, (1, 72, 24, 24)).to(dev))
y3 = _ext.dcn_v2_forward(x, w, b, off, msk, 3, 3, 1, 1, 1, 1, 1, 1, 8)
mp = ops.psa_maxpool2(xp)
yi = ops.dcn_v2_fused_tc(xp, om, w, b, 8)
back = ops.psa_to_f32(a)
# grouped deformable convolution, v1 and modulated, fp32 and fp64, forward and backward (3 conv groups of 4 input
# channels against 2 deformable groups of 6, Cout_g = 7: a partial NO block)
from mmsr.models.archs.dcn import deform_conv, modulated_deform_conv
for dt in (torch.float32, torch.float64):
    xg = seeding.randn(10, (2, 12, 9, 11)).to(dev, dt).requires_grad_(True)
    wg = seeding.randn(11, (21, 4, 3, 3), 0.2).to(dev, dt).requires_grad_(True)
    og = seeding.randn(12, (2, 36, 9, 11), 2.0).to(dev, dt).requires_grad_(True)
    mg = torch.sigmoid(seeding.randn(13, (2, 18, 9, 11))).to(dev, dt).requires_grad_(True)
    deform_conv(xg, og, wg, 1, 1, 1, 3, 2).sum().backward()
    modulated_deform_conv(xg, og, mg, wg, None, 1, 1, 1, 3, 2).sum().backward()
# a search that overflows its candidate lists (constant features: every score ties) -> exhaustive re-scan kernels
flat = torch.ones(1, 64, 20, 22, device=dev)
os.environ['C2M_CORR_EXACT_TIES'] = '1'          # no budget: the exhaustive pass must run under the sanitizer
c2m.corr_argmax(flat, flat, norm_input=True, l2norm=True)
os.environ.pop('C2M_CORR_EXACT_TIES')
torch.cuda.synchronize()
print('ok', float((y1 - y2).abs().max()), tuple(d.shape), tuple(e.shape))
