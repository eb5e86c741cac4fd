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
// Sampling points, corners and the shape check are the forward's (dcn_sampling.cuh); a corner
// outside the image is skipped here, where the forward loads element 0 with weight 0.
//
// The kernels are templated on the scalar type and also serve `deform_conv_cuda` (mmsr/models/archs/dcn):
// a null mask is a modulation of 1 and then no grad_mask is written.  The reference's DCNv1 kernels
// (deformable_im2col / col2im / col2im_coord, dcn/src/deform_conv_cuda_kernel.cu:116-434) are these formulas with
// m = 1, and their 5x5-window scatter reaches the same <= 4 corners.  Conv groups enter only the two GEMMs.
#include "dcn_sampling.cuh"

namespace c2m {

// one thread per (b, c, p): all taps
template <typename scalar_t>
__global__ void dcn_im2col_kernel(const scalar_t *__restrict__ x, const scalar_t *__restrict__ offset,
                                  const scalar_t *__restrict__ mask, const c2m_dcn_shape s, const DcnGeom d,
                                  scalar_t *__restrict__ col) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.C * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), c = (int)((e / P) % s.C), b = (int)(e / ((long long)P * s.C));
        const int grp = c / cpg;
        const scalar_t *im = x + ((long long)b * s.C + c) * s.H * s.W;
        for (int k = 0; k < T; ++k) {
            const long long j = ((long long)b * s.dg + grp) * T + k;   // (image, group, tap) plane
            scalar_t h_im, w_im, v = 0;
            if (dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) {
                const DcnCorners<scalar_t> q(h_im, w_im, s.H, s.W, s.W, 1);
                const scalar_t v1 = q.ok[0] ? im[q.o[0]] : (scalar_t)0, v2 = q.ok[1] ? im[q.o[1]] : (scalar_t)0;
                const scalar_t v3 = q.ok[2] ? im[q.o[2]] : (scalar_t)0, v4 = q.ok[3] ? im[q.o[3]] : (scalar_t)0;
                v = dcn_blend(q.w, v1, v2, v3, v4) * (mask ? mask[j * P + p] : (scalar_t)1);
            }
            col[((long long)b * s.C * T + (long long)c * T + k) * P + p] = v;
        }
    }
}

// one thread per (b, group, tap, p): reduce over the group's channels
template <typename scalar_t>
__global__ void dcn_col2im_coord_kernel(const scalar_t *__restrict__ gcol, const scalar_t *__restrict__ x,
                                        const scalar_t *__restrict__ offset, const scalar_t *__restrict__ mask,
                                        const c2m_dcn_shape s, const DcnGeom d, scalar_t *__restrict__ goff,
                                        scalar_t *__restrict__ gmask) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.dg * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), grp = (int)((e / ((long long)P * T)) % s.dg);
        const int b = (int)(e / ((long long)P * T * s.dg));
        const long long j = ((long long)b * s.dg + grp) * T + k;
        scalar_t h_im, w_im;
        scalar_t acc_h = 0, acc_w = 0, acc_m = 0;
        if (dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) {
            const scalar_t m = mask ? mask[j * P + p] : (scalar_t)1;
            const DcnCorners<scalar_t> q(h_im, w_im, s.H, s.W, s.W, 1);
            const scalar_t hh = (scalar_t)1 - q.lh, hw = (scalar_t)1 - q.lw;
            for (int cl = 0; cl < cpg; ++cl) {
                const int c = grp * cpg + cl;
                const scalar_t gc = gcol[((long long)b * s.C * T + (long long)c * T + k) * P + p];
                const scalar_t *im = x + ((long long)b * s.C + c) * s.H * s.W;
                const scalar_t v1 = q.ok[0] ? im[q.o[0]] : (scalar_t)0, v2 = q.ok[1] ? im[q.o[1]] : (scalar_t)0;
                const scalar_t v3 = q.ok[2] ? im[q.o[2]] : (scalar_t)0, v4 = q.ok[3] ? im[q.o[3]] : (scalar_t)0;
                acc_m += gc * dcn_blend(q.w, v1, v2, v3, v4);
                acc_h += gc * m * (-hw * v1 - q.lw * v2 + hw * v3 + q.lw * v4);
                acc_w += gc * m * (-hh * v1 + hh * v2 - q.lh * v3 + q.lh * v4);
            }
        }
        goff[2 * j * P + p] = acc_h;
        goff[(2 * j + 1) * P + p] = acc_w;
        if (gmask) gmask[j * P + p] = acc_m;
    }
}

// one thread per (b, c, tap, p): scatter to the contributing corners
template <typename scalar_t>
__global__ void dcn_col2im_kernel(const scalar_t *__restrict__ gcol, const scalar_t *__restrict__ offset,
                                  const scalar_t *__restrict__ mask, const c2m_dcn_shape s, const DcnGeom d,
                                  scalar_t *__restrict__ gx) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.C * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), c = (int)((e / ((long long)P * T)) % s.C);
        const int b = (int)(e / ((long long)P * T * s.C));
        const long long j = ((long long)b * s.dg + c / cpg) * T + k;
        scalar_t h_im, w_im;
        if (!dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) continue;
        const scalar_t tg = gcol[e] * (mask ? mask[j * P + p] : (scalar_t)1);
        const DcnCorners<scalar_t> q(h_im, w_im, s.H, s.W, s.W, 1);
        const scalar_t hh = (scalar_t)1 - q.lh, hw = (scalar_t)1 - q.lw;
        scalar_t *gim = gx + ((long long)b * s.C + c) * s.H * s.W;
        if (q.ok[0]) atomicAdd(gim + q.o[0], tg * hh * hw);
        if (q.ok[1]) atomicAdd(gim + q.o[1], tg * hh * q.lw);
        if (q.ok[2]) atomicAdd(gim + q.o[2], tg * q.lh * hw);
        if (q.ok[3]) atomicAdd(gim + q.o[3], tg * q.lh * q.lw);
    }
}

static inline int blocks_for(long long n) { long long b = (n + 255) / 256; return (int)(b > 132 * 16 ? 132 * 16 : b); }

template <typename scalar_t>
static int im2col(const scalar_t *x, const scalar_t *offset, const scalar_t *mask, const c2m_dcn_shape *shape,
                  scalar_t *columns, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_im2col_kernel<<<blocks_for((long long)shape->B * shape->C * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(x, offset, mask, *shape, d, columns);
    C2M_LAUNCH_CHECK("dcn_im2col_kernel");
    return C2M_OK;
}

template <typename scalar_t>
static int col2im_coord(const scalar_t *gcol, const scalar_t *x, const scalar_t *offset, const scalar_t *mask,
                        const c2m_dcn_shape *shape, scalar_t *grad_offset, scalar_t *grad_mask, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_col2im_coord_kernel<<<blocks_for((long long)shape->B * shape->dg * d.T * d.Ho * d.Wo), 256, 0,
                              reinterpret_cast<cudaStream_t>(stream)>>>(gcol, x, offset, mask, *shape, d, grad_offset,
                                                                        grad_mask);
    C2M_LAUNCH_CHECK("dcn_col2im_coord_kernel");
    return C2M_OK;
}

template <typename scalar_t>
static int col2im(const scalar_t *gcol, const scalar_t *offset, const scalar_t *mask, const c2m_dcn_shape *shape,
                  scalar_t *grad_input, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_col2im_kernel<<<blocks_for((long long)shape->B * shape->C * d.T * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(gcol, offset, mask, *shape, d, grad_input);
    C2M_LAUNCH_CHECK("dcn_col2im_kernel");
    return C2M_OK;
}

}  // namespace c2m

using namespace c2m;

extern "C" int c2m_dcn_v2_im2col_f32(const float *x, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *columns, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && mask && columns, "dcn_v2_im2col: null pointer");
    return im2col(x, offset, mask, shape, columns, stream);
}

extern "C" int c2m_dcn_v2_col2im_coord_f32(const float *gcol, const float *x, const float *offset, const float *mask,
                                           const c2m_dcn_shape *shape, float *grad_offset, float *grad_mask,
                                           c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && x && offset && mask && grad_offset && grad_mask, "dcn_v2_col2im_coord: null pointer");
    return col2im_coord(gcol, x, offset, mask, shape, grad_offset, grad_mask, stream);
}

extern "C" int c2m_dcn_v2_col2im_f32(const float *gcol, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *grad_input, c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && offset && mask && grad_input, "dcn_v2_col2im: null pointer");
    return col2im(gcol, offset, mask, shape, grad_input, stream);
}

// deform_conv_cuda: mask may be NULL (DCNv1), and grad_mask is NULL exactly when mask is
#define C2M_DEFORM_CONV_BWD(T, SFX)                                                                                 \
    extern "C" int c2m_deform_conv_im2col_##SFX(const T *x, const T *offset, const T *mask,                         \
                                                const c2m_dcn_shape *shape, T *columns, c2m_stream_t stream) {      \
        C2M_CHECK_ARG(x && offset && columns, "deform_conv_im2col: null pointer");                                  \
        return im2col(x, offset, mask, shape, columns, stream);                                                     \
    }                                                                                                               \
    extern "C" int c2m_deform_conv_col2im_coord_##SFX(const T *gcol, const T *x, const T *offset, const T *mask,    \
                                                      const c2m_dcn_shape *shape, T *grad_offset, T *grad_mask,     \
                                                      c2m_stream_t stream) {                                        \
        C2M_CHECK_ARG(gcol && x && offset && grad_offset, "deform_conv_col2im_coord: null pointer");                \
        C2M_CHECK_ARG((mask == nullptr) == (grad_mask == nullptr),                                                  \
                      "deform_conv_col2im_coord: grad_mask must be given exactly when mask is");                    \
        return col2im_coord(gcol, x, offset, mask, shape, grad_offset, grad_mask, stream);                          \
    }                                                                                                               \
    extern "C" int c2m_deform_conv_col2im_##SFX(const T *gcol, const T *offset, const T *mask,                      \
                                                const c2m_dcn_shape *shape, T *grad_input, c2m_stream_t stream) {   \
        C2M_CHECK_ARG(gcol && offset && grad_input, "deform_conv_col2im: null pointer");                            \
        return col2im(gcol, offset, mask, shape, grad_input, stream);                                               \
    }

C2M_DEFORM_CONV_BWD(float, f32)
C2M_DEFORM_CONV_BWD(double, f64)
