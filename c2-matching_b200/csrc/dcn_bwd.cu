// DCNv2 backward building blocks (SURVEY.md §8f N4; completes the `_ext` ABI:
// `_ext.dcn_v2_backward`, DCNv2/src/dcn_v2.h:41-72, dcn_v2_cuda.cu:206-335).
//
// Training is not on the restoration-forward hot path, so this keeps the reference's
// decomposition — column-gradient GEMM, coordinate/mask gradient, input-gradient scatter, column
// matrix for the weight gradient — with the two dense GEMMs left to the caller (torch.matmul) and
// the three deformable pieces written here:
//   c2m_dcn_v2_im2col_f32        columns[b, c*T+k, p] = mask * bilinear(x)          (:125-195)
//   c2m_dcn_v2_col2im_coord_f32  grad_offset / grad_mask from gcol                   (:256-327, 83-123)
//   c2m_dcn_v2_col2im_f32        grad_input += scatter of gcol * mask                (:197-254, 56-80)
// Unlike the reference, batch is a grid dimension (no host loop), grad_input scatter touches only
// the (<= 4) contributing corners instead of a 5x5 window, and launch errors are returned.
#include "c2m_common.cuh"

namespace c2m {

namespace {
struct Geo {
    int B, C, H, W, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
};

__device__ __forceinline__ bool sample_pos(const Geo &g, const float *offset, int b, int grp, int k, int p, float &h_im,
                                           float &w_im) {
    const int T = g.kh * g.kw, P = g.Ho * g.Wo;
    const int ho = p / g.Wo, wo = p % g.Wo, i = k / g.kw, j = k % g.kw;
    const float oh = offset[(((long long)b * g.dg + grp) * 2 * T + 2 * k) * P + p];
    const float ow = offset[(((long long)b * g.dg + grp) * 2 * T + 2 * k + 1) * P + p];
    h_im = (float)(ho * g.sh - g.ph + i * g.dh) + oh;
    w_im = (float)(wo * g.sw - g.pw + j * g.dw) + ow;
    return h_im > -1.f && w_im > -1.f && h_im < (float)g.H && w_im < (float)g.W;
}
}  // namespace

// one thread per (b, c, p): 9 taps
__global__ void dcn_im2col_kernel(const float *__restrict__ x, const float *__restrict__ offset,
                                  const float *__restrict__ mask, Geo g, float *__restrict__ col) {
    const int T = g.kh * g.kw, P = g.Ho * g.Wo, cpg = g.C / g.dg;
    const long long n = (long long)g.B * g.C * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), c = (int)((e / P) % g.C), b = (int)(e / ((long long)P * g.C));
        const int grp = c / cpg;
        const float *im = x + ((long long)b * g.C + c) * g.H * g.W;
        for (int k = 0; k < T; ++k) {
            float h_im, w_im, v = 0.f;
            if (sample_pos(g, offset, b, grp, k, p, h_im, w_im)) {
                const int hl = (int)floorf(h_im), wl = (int)floorf(w_im), hh = hl + 1, wh = wl + 1;
                const float lh = h_im - hl, lw = w_im - wl, uh = 1.f - lh, uw = 1.f - lw;
                float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
                if (hl >= 0 && wl >= 0) v1 = im[hl * g.W + wl];
                if (hl >= 0 && wh <= g.W - 1) v2 = im[hl * g.W + wh];
                if (hh <= g.H - 1 && wl >= 0) v3 = im[hh * g.W + wl];
                if (hh <= g.H - 1 && wh <= g.W - 1) v4 = im[hh * g.W + wh];
                v = (uh * uw * v1 + uh * lw * v2 + lh * uw * v3 + lh * lw * v4) *
                    mask[(((long long)b * g.dg + grp) * T + k) * P + p];
            }
            col[((long long)b * g.C * T + (long long)c * T + k) * P + p] = v;
        }
    }
}

// one thread per (b, group, tap, p): reduce over the group's channels
__global__ void dcn_col2im_coord_kernel(const float *__restrict__ gcol, const float *__restrict__ x,
                                        const float *__restrict__ offset, const float *__restrict__ mask, Geo g,
                                        float *__restrict__ goff, float *__restrict__ gmask) {
    const int T = g.kh * g.kw, P = g.Ho * g.Wo, cpg = g.C / g.dg;
    const long long n = (long long)g.B * g.dg * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), grp = (int)((e / ((long long)P * T)) % g.dg);
        const int b = (int)(e / ((long long)P * T * g.dg));
        float h_im, w_im;
        float acc_h = 0.f, acc_w = 0.f, acc_m = 0.f;
        if (sample_pos(g, offset, b, grp, k, p, h_im, w_im)) {
            const float m = mask[(((long long)b * g.dg + grp) * T + k) * P + p];
            const int hl = (int)floorf(h_im), wl = (int)floorf(w_im), hh = hl + 1, wh = wl + 1;
            const float lh = h_im - hl, lw = w_im - wl, uh = 1.f - lh, uw = 1.f - lw;
            const bool c1 = hl >= 0 && wl >= 0, c2 = hl >= 0 && wh <= g.W - 1, c3 = hh <= g.H - 1 && wl >= 0,
                       c4 = hh <= g.H - 1 && wh <= g.W - 1;
            for (int cl = 0; cl < cpg; ++cl) {
                const int c = grp * cpg + cl;
                const float gc = gcol[((long long)b * g.C * T + (long long)c * T + k) * P + p];
                const float *im = x + ((long long)b * g.C + c) * g.H * g.W;
                const float v1 = c1 ? im[hl * g.W + wl] : 0.f, v2 = c2 ? im[hl * g.W + wh] : 0.f;
                const float v3 = c3 ? im[hh * g.W + wl] : 0.f, v4 = c4 ? im[hh * g.W + wh] : 0.f;
                acc_m += gc * (uh * uw * v1 + uh * lw * v2 + lh * uw * v3 + lh * lw * v4);
                acc_h += gc * m * (-uw * v1 - lw * v2 + uw * v3 + lw * v4);
                acc_w += gc * m * (-uh * v1 + uh * v2 - lh * v3 + lh * v4);
            }
        }
        goff[(((long long)b * g.dg + grp) * 2 * T + 2 * k) * P + p] = acc_h;
        goff[(((long long)b * g.dg + grp) * 2 * T + 2 * k + 1) * P + p] = acc_w;
        gmask[(((long long)b * g.dg + grp) * T + k) * P + p] = acc_m;
    }
}

// one thread per (b, c, tap, p): scatter to the contributing corners
__global__ void dcn_col2im_kernel(const float *__restrict__ gcol, const float *__restrict__ offset,
                                  const float *__restrict__ mask, Geo g, float *__restrict__ gx) {
    const int T = g.kh * g.kw, P = g.Ho * g.Wo, cpg = g.C / g.dg;
    const long long n = (long long)g.B * g.C * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), c = (int)((e / ((long long)P * T)) % g.C);
        const int b = (int)(e / ((long long)P * T * g.C));
        const int grp = c / cpg;
        float h_im, w_im;
        if (!sample_pos(g, offset, b, grp, k, p, h_im, w_im)) continue;
        const float tg = gcol[e] * mask[(((long long)b * g.dg + grp) * T + k) * P + p];
        const int hl = (int)floorf(h_im), wl = (int)floorf(w_im), hh = hl + 1, wh = wl + 1;
        const float lh = h_im - hl, lw = w_im - wl, uh = 1.f - lh, uw = 1.f - lw;
        float *gim = gx + ((long long)b * g.C + c) * g.H * g.W;
        if (hl >= 0 && wl >= 0) atomicAdd(gim + hl * g.W + wl, tg * uh * uw);
        if (hl >= 0 && wh <= g.W - 1) atomicAdd(gim + hl * g.W + wh, tg * uh * lw);
        if (hh <= g.H - 1 && wl >= 0) atomicAdd(gim + hh * g.W + wl, tg * lh * uw);
        if (hh <= g.H - 1 && wh <= g.W - 1) atomicAdd(gim + hh * g.W + wh, tg * lh * lw);
    }
}

static int make_geo(Geo &g, const c2m_dcn_shape *s) {
    C2M_CHECK_ARG(s, "dcn backward: null shape");
    C2M_CHECK_ARG(s->B > 0 && s->C > 0 && s->H > 0 && s->W > 0, "dcn backward: empty tensor");
    C2M_CHECK_ARG(s->kh > 0 && s->kw > 0 && s->sh > 0 && s->sw > 0 && s->dh > 0 && s->dw > 0, "dcn backward: bad kernel geometry");
    C2M_CHECK_ARG(s->dg > 0 && s->C % s->dg == 0, "dcn backward: channels (%d) not divisible by deformable_group (%d)", s->C, s->dg);
    g = Geo{s->B, s->C, s->H, s->W, s->kh, s->kw, s->sh, s->sw, s->ph, s->pw, s->dh, s->dw, s->dg, 0, 0};
    g.Ho = (s->H + 2 * s->ph - (s->dh * (s->kh - 1) + 1)) / s->sh + 1;
    g.Wo = (s->W + 2 * s->pw - (s->dw * (s->kw - 1) + 1)) / s->sw + 1;
    C2M_CHECK_ARG(g.Ho > 0 && g.Wo > 0, "dcn backward: empty output");
    return C2M_OK;
}
static inline int blocks_for(long long n) { long long b = (n + 255) / 256; return (int)(b > 132 * 16 ? 132 * 16 : b); }

}  // namespace c2m

using namespace c2m;

extern "C" int c2m_dcn_v2_im2col_f32(const float *x, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *columns, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && mask && columns, "dcn_v2_im2col: null pointer");
    Geo g;
    if (int rc = make_geo(g, shape)) return rc;
    dcn_im2col_kernel<<<blocks_for((long long)g.B * g.C * g.Ho * g.Wo), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        x, offset, mask, g, columns);
    C2M_LAUNCH_CHECK("dcn_im2col_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_v2_col2im_coord_f32(const float *gcol, const float *x, const float *offset, const float *mask,
                                           const c2m_dcn_shape *shape, float *grad_offset, float *grad_mask,
                                           c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && x && offset && mask && grad_offset && grad_mask, "dcn_v2_col2im_coord: null pointer");
    Geo g;
    if (int rc = make_geo(g, shape)) return rc;
    dcn_col2im_coord_kernel<<<blocks_for((long long)g.B * g.dg * g.kh * g.kw * g.Ho * g.Wo), 256, 0,
                              reinterpret_cast<cudaStream_t>(stream)>>>(gcol, x, offset, mask, g, grad_offset, grad_mask);
    C2M_LAUNCH_CHECK("dcn_col2im_coord_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_v2_col2im_f32(const float *gcol, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *grad_input, c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && offset && mask && grad_input, "dcn_v2_col2im: null pointer");
    Geo g;
    if (int rc = make_geo(g, shape)) return rc;
    dcn_col2im_kernel<<<blocks_for((long long)g.B * g.C * g.kh * g.kw * g.Ho * g.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(gcol, offset, mask, g, grad_input);
    C2M_LAUNCH_CHECK("dcn_col2im_kernel");
    return C2M_OK;
}
