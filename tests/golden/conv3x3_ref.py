"""fp64 reference of the 3x3 / stride 1 / pad 1 convolution and its gradients, written as nine explicit shifted-slice
products with broadcasting (no BLAS, so no library decides how 0 * Inf or NaN enters a sum).

Non-finite semantics follow torch's fp64 CPU functions:
  forward  out[p] = b + sum over taps of w[tap] . xpad[p + tap]          x zero-padded: a non-finite weight meets the
                                                                         padding's zeros (0 * Inf = NaN), as F.conv2d
  dX       dX[q]  = sum over in-map p, tap with p + tap - 1 = q of w[tap]^T gy[p]
                                                                         (scattered: no pixel outside the map takes
                                                                         part, as torch.nn.grad.conv2d_input)
  dW       dW[tap] = sum over in-map p of gy[p] xpad[p + tap]^T           (x zero-padded, as conv2d_weight)
  db       plain sum of gy over batch and pixels.
Every function runs on the tensors' device; chunked so that no broadcast product exceeds CHUNK elements."""
import torch

CHUNK = 1 << 24


def _chunks(n, per):
    step = max(1, CHUNK // max(1, per))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def _pad(t):
    return torch.nn.functional.pad(t, (1, 1, 1, 1))


def conv3x3_forward(x, w, b=None):
    """x [B,Cin,H,W], w [Cout,Cin,3,3], b [Cout] or None -> out [B,Cout,H,W] in fp64."""
    x, w = x.double(), w.double()
    B, cin, H, W = x.shape
    cout = w.shape[0]
    xp = _pad(x)
    out = torch.zeros(B, cout, H, W, dtype=torch.float64, device=x.device)
    for ky in range(3):
        for kx in range(3):
            xs = xp[:, :, ky:ky + H, kx:kx + W]                         # [B,Cin,H,W]
            wt = w[:, :, ky, kx]                                        # [Cout,Cin]
            for bi in range(B):
                for c0, c1 in _chunks(cout, cin * H * W):
                    out[bi, c0:c1] += (wt[c0:c1, :, None, None] * xs[bi][None]).sum(1)
    if b is not None:
        out += b.double()[None, :, None, None]
    return out


def conv3x3_grad_input(w, gy):
    """dX [B,Cin,H,W] of the convolution above for grad_output gy [B,Cout,H,W], fp64."""
    w, gy = w.double(), gy.double()
    B, cout, H, W = gy.shape
    cin = w.shape[1]
    dxp = torch.zeros(B, cin, H + 2, W + 2, dtype=torch.float64, device=gy.device)
    for ky in range(3):
        for kx in range(3):
            wt = w[:, :, ky, kx]                                        # [Cout,Cin]
            for bi in range(B):
                for c0, c1 in _chunks(cin, cout * H * W):
                    dxp[bi, c0:c1, ky:ky + H, kx:kx + W] += (wt[:, c0:c1, None, None] * gy[bi][:, None]).sum(0)
    return dxp[:, :, 1:H + 1, 1:W + 1].contiguous()


def conv3x3_grad_weight(x, gy):
    """dW [Cout,Cin,3,3] for input x [B,Cin,H,W] and grad_output gy [B,Cout,H,W], fp64."""
    x, gy = x.double(), gy.double()
    B, cin, H, W = x.shape
    cout = gy.shape[1]
    xp = _pad(x)
    dw = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device=x.device)
    for ky in range(3):
        for kx in range(3):
            xs = xp[:, :, ky:ky + H, kx:kx + W]
            for bi in range(B):
                for c0, c1 in _chunks(cout, cin * H * W):
                    dw[c0:c1, :, ky, kx] += (gy[bi, c0:c1, None] * xs[bi][None]).sum((2, 3))
    return dw


def conv3x3_grads(x, w, gy):
    """(dX, dW, db) in fp64."""
    return conv3x3_grad_input(w, gy), conv3x3_grad_weight(x, gy), gy.double().sum((0, 2, 3))
