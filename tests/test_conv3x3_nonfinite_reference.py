"""CPU checks of the fp64 3x3-convolution reference (tests/golden/conv3x3_ref.py) that the range and non-finite tests of
the tensor-core convolution (test_gpu_conv3x3_range.py) compare against: its values equal torch's fp64 convolution and
gradients on finite inputs, its finiteness pattern equals theirs for NaN / +-Inf in x, the weights and grad_output at
the placements the GPU tests use, and a small case worked out by hand, including an Inf in the last row of a map whose
height is not a multiple of the 16-row tile, comes out as expected."""
import pytest
import torch
import torch.nn.functional as F

import conv3x3_ref as R


def _torch(x, w, b, gy):
    return (F.conv2d(x, w, b, 1, 1), torch.nn.grad.conv2d_input(x.shape, w, gy, 1, 1),
            torch.nn.grad.conv2d_weight(x, w.shape, gy, 1, 1), gy.sum((0, 2, 3)))


def _ref(x, w, b, gy):
    return (R.conv3x3_forward(x, w, b),) + R.conv3x3_grads(x, w, gy)


def _case(seed, B, cin, cout, H, W):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, cin, H, W, generator=g, dtype=torch.float64),
            torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64),
            torch.randn(cout, generator=g, dtype=torch.float64),
            torch.randn(B, cout, H, W, generator=g, dtype=torch.float64))


@pytest.mark.parametrize('shape', [(2, 5, 4, 9, 7), (1, 3, 8, 21, 13), (2, 16, 12, 19, 11), (1, 1, 1, 3, 3)])
def test_reference_equals_torch_fp64_on_finite_inputs(shape):
    x, w, b, gy = _case(1, *shape)
    for name, want, got in zip(('out', 'dX', 'dW', 'db'), _torch(x, w, b, gy), _ref(x, w, b, gy)):
        assert float((want - got).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max())), name


# the placements of test_gpu_conv3x3_range.py: corners, last row / column at the middle, an interior pixel
def _pixels(H, W):
    return [(0, 0), (H - 1, W - 1), (H - 1, W // 2), (H // 2, W - 1), (H // 3, W // 3)]


@pytest.mark.parametrize('bad', ['nan', 'inf', '-inf'])
@pytest.mark.parametrize('hw', [(21, 13), (19, 11), (32, 16)])
def test_nonfinite_pattern_equals_torch_fp64(bad, hw):
    H, W = hw
    x, w, b, gy = _case(2, 2, 6, 5, H, W)
    for where in ('x', 'gy'):
        for y, xx in _pixels(H, W):
            xs, gs = x.clone(), gy.clone()
            (xs if where == 'x' else gs)[1, 3 if where == 'x' else 2, y, xx] = float(bad)
            for name, want, got in zip(('out', 'dX', 'dW', 'db'), _torch(xs, w, b, gs), _ref(xs, w, b, gs)):
                assert torch.equal(torch.isfinite(want), torch.isfinite(got)), (where, y, xx, name)
    for tap in range(9):
        ws = w.clone()
        ws[2, 4, tap // 3, tap % 3] = float(bad)
        for name, want, got in zip(('out', 'dX', 'dW', 'db'), _torch(x, ws, b, gy), _ref(x, ws, b, gy)):
            assert torch.equal(torch.isfinite(want), torch.isfinite(got)), ('w', tap, name)


def test_small_case_by_hand():
    """One channel, 3 x 3 map, all-ones weights: out is the 3 x 3 box sum of the zero-padded x plus the bias, dX of an
    all-ones gradient counts the in-map neighbours, dW[tap] sums the x pixels the tap reaches."""
    x = torch.arange(1., 10., dtype=torch.float64).view(1, 1, 3, 3)
    w = torch.ones(1, 1, 3, 3, dtype=torch.float64)
    out = R.conv3x3_forward(x, w, torch.tensor([0.5], dtype=torch.float64))
    assert out[0, 0].tolist() == [[12.5, 21.5, 16.5], [27.5, 45.5, 33.5], [24.5, 39.5, 28.5]]
    gy = torch.ones(1, 1, 3, 3, dtype=torch.float64)
    dx, dw, db = R.conv3x3_grads(x, w, gy)
    assert dx[0, 0].tolist() == [[4., 6., 4.], [6., 9., 6.], [4., 6., 4.]]
    # tap (ky, kx) pairs output p with x[p + (ky - 1, kx - 1)]: the corner taps see a 2 x 2 block of x
    assert dw[0, 0].tolist() == [[12., 21., 16.], [27., 45., 33.], [24., 39., 28.]]
    assert db.tolist() == [9.]


def test_ragged_last_row_keeps_the_top_taps_finite():
    """Inf at (H-1, c) of a 19 x 11 map (19 % 16 != 0): only the output pixels at rows H-2 and H-1 (and the last row's
    zero-padded neighbour, which is not an output) see it.  dW[ky = 0] pairs output row y with x row y - 1, which
    reaches row H-1 only from output row H, outside the map, so the three ky = 0 taps stay finite; the six others do
    not.  A corner Inf at (0, 0) leaves the five taps with ky = 2 or kx = 2 finite."""
    H, W = 19, 11
    x, w, b, gy = _case(3, 1, 1, 1, H, W)
    xs = x.clone()
    xs[0, 0, H - 1, 5] = float('inf')
    fin = torch.isfinite(R.conv3x3_grad_weight(xs, gy))[0, 0]
    assert fin.tolist() == [[True] * 3, [False] * 3, [False] * 3]
    xs = x.clone()
    xs[0, 0, 7, W - 1] = float('inf')
    assert torch.isfinite(R.conv3x3_grad_weight(xs, gy))[0, 0].tolist() == [[True, False, False]] * 3
    xs = x.clone()
    xs[0, 0, H - 1, W - 1] = float('inf')
    assert int(torch.isfinite(R.conv3x3_grad_weight(xs, gy)).sum()) == 5
    xs = x.clone()
    xs[0, 0, 0, 0] = float('inf')
    assert torch.isfinite(R.conv3x3_grad_weight(xs, gy))[0, 0].tolist() == [[False, False, True], [False, False, True],
                                                                             [True, True, True]]
    # the forward: the nine output pixels around the Inf are non-finite, every other one is finite
    xs = x.clone()
    xs[0, 0, H - 1, 5] = float('inf')
    out = torch.isfinite(R.conv3x3_forward(xs, w, b))[0, 0]
    assert int((~out).sum()) == 6 and not bool(out[H - 2:, 4:7].any())
