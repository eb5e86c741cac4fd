// The deformable sampling rule of the CUDA-core DCN kernels (dcn_v2.cu, dcn_bwd.cu) and the index-map
// decode (offsets.cu), stated once.  Arithmetic follows dmcn_im2col_bilinear (dcn_v2_im2col_cuda.cu:25-54,
// 125-195) operation for operation; keep each expression's order, the kernels' results depend on it bit for bit.
// The sampling rule is templated on the scalar type: float serves `_ext` and both dtypes serve deform_conv_cuda.
#pragma once
#include "c2m_common.cuh"

namespace c2m {

struct DcnGeom { int Ho, Wo, T, cpg; };   // output size, taps (kh * kw), channels per deformable group

// Checks `s` and derives `g`; error messages start with `who`.
static inline int dcn_geometry(const c2m_dcn_shape *s, const char *who, DcnGeom &g) {
    C2M_CHECK_ARG(s, "%s: null shape", who);
    C2M_CHECK_ARG(s->B > 0 && s->C > 0 && s->H > 0 && s->W > 0, "%s: empty tensor", who);
    C2M_CHECK_ARG(s->kh > 0 && s->kw > 0 && s->sh > 0 && s->sw > 0 && s->dh > 0 && s->dw > 0, "%s: bad kernel geometry", who);
    C2M_CHECK_ARG(s->dg > 0 && s->C % s->dg == 0, "%s: channels (%d) not divisible by deformable_group (%d)", who, s->C, s->dg);
    g.Ho = (s->H + 2 * s->ph - (s->dh * (s->kh - 1) + 1)) / s->sh + 1;
    g.Wo = (s->W + 2 * s->pw - (s->dw * (s->kw - 1) + 1)) / s->sw + 1;
    C2M_CHECK_ARG(g.Ho > 0 && g.Wo > 0, "%s: empty output (%d x %d)", who, g.Ho, g.Wo);
    g.T = s->kh * s->kw;
    g.cpg = s->C / s->dg;
    return C2M_OK;
}

// Sampling point of tap k at output pixel p (row-major, Wo wide) moved by the final offset (off_h, off_w);
// false outside -1 < h < H, -1 < w < W, where the sample is 0.  T is the scalar type (float or double) positions are
// computed in, as the reference's `scalar_t` kernels do.
template <typename T>
__device__ __forceinline__ bool dcn_sample_point(const c2m_dcn_shape &s, int Wo, int k, int p, T off_h, T off_w,
                                                 T &h_im, T &w_im) {
    const int ho = p / Wo, wo = p % Wo, i = k / s.kw, j = k % s.kw;
    h_im = (T)(ho * s.sh - s.ph + i * s.dh) + off_h;
    w_im = (T)(wo * s.sw - s.pw + j * s.dw) + off_w;
    return h_im > (T)-1 && w_im > (T)-1 && h_im < (T)s.H && w_im < (T)s.W;
}

template <typename T>
__device__ __forceinline__ T dcn_blend(const T (&w)[4], T v0, T v1, T v2, T v3) {
    return w[0] * v0 + w[1] * v1 + w[2] * v2 + w[3] * v3;
}

__device__ __forceinline__ float dcn_floor(float v) { return floorf(v); }
__device__ __forceinline__ double dcn_floor(double v) { return floor(v); }

// Bilinear corners (low, low), (low, high), (high, low), (high, high) in (row, column) of an in-window point;
// a corner outside the image is not `ok`.  Offsets are row * ys + column * xs.
template <typename T>
struct DcnCorners {
    bool ok[4];
    T w[4];         // hh*hw, hh*lw, lh*hw, lh*lw with hh = 1 - lh, hw = 1 - lw
    T lh, lw;
    int o[4];

    template <typename S>
    __device__ __forceinline__ DcnCorners(T h_im, T w_im, int H, int W, S ys, S xs) {
        const int h_low = (int)dcn_floor(h_im), w_low = (int)dcn_floor(w_im);
        const int h_high = h_low + 1, w_high = w_low + 1;
        lh = h_im - h_low;
        lw = w_im - w_low;
        const T hh = (T)1 - lh, hw = (T)1 - lw;
        const bool t0 = h_low >= 0, t1 = h_high <= H - 1, l0 = w_low >= 0, l1 = w_high <= W - 1;
        ok[0] = t0 && l0; w[0] = hh * hw; o[0] = (int)(h_low * ys + w_low * xs);
        ok[1] = t0 && l1; w[1] = hh * lw; o[1] = (int)(h_low * ys + w_high * xs);
        ok[2] = t1 && l0; w[2] = lh * hw; o[2] = (int)(h_high * ys + w_low * xs);
        ok[3] = t1 && l1; w[3] = lh * lw; o[3] = (int)(h_high * ys + w_high * xs);
    }
};

// Flow (x, y) of tap (i, j) of the scale-s pre-offset pyramid at (Y, X) of image b, decoded from the index-map
// cell the tap shifts there; 0 off the map (index_to_flow + tensor_shift, corres_generation_arch.py:29-104).
__device__ __forceinline__ float2 pyramid_flow(const long long *idx, int b, int gh, int gw, int ref_gw, int s, int Y,
                                               int X, int i, int j) {
    float2 f = make_float2(0.f, 0.f);
    const int ys = Y - s * i, xs = X - s * j;
    if (ys >= 0 && xs >= 0) {
        const int y = ys / s, x = xs / s;
        if (y < gh && x < gw) {
            const long long v = idx[((long long)b * gh + y) * gw + x];
            f.x = (float)(s * ((int)(v % ref_gw) - x));
            f.y = (float)(s * ((int)(v / ref_gw) - y));
        }
    }
    return f;
}

}  // namespace c2m
