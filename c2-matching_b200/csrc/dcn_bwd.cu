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
#include "dcn_sampling.cuh"

namespace c2m {

// one thread per (b, c, p): all taps
__global__ void dcn_im2col_kernel(const float *__restrict__ x, const float *__restrict__ offset,
                                  const float *__restrict__ mask, const c2m_dcn_shape s, const DcnGeom d,
                                  float *__restrict__ col) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.C * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), c = (int)((e / P) % s.C), b = (int)(e / ((long long)P * s.C));
        const int grp = c / cpg;
        const float *im = x + ((long long)b * s.C + c) * s.H * s.W;
        for (int k = 0; k < T; ++k) {
            const long long j = ((long long)b * s.dg + grp) * T + k;   // (image, group, tap) plane
            float h_im, w_im, v = 0.f;
            if (dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) {
                const DcnCorners q(h_im, w_im, s.H, s.W, s.W, 1);
                const float v1 = q.ok[0] ? im[q.o[0]] : 0.f, v2 = q.ok[1] ? im[q.o[1]] : 0.f;
                const float v3 = q.ok[2] ? im[q.o[2]] : 0.f, v4 = q.ok[3] ? im[q.o[3]] : 0.f;
                v = dcn_blend(q.w, v1, v2, v3, v4) * mask[j * P + p];
            }
            col[((long long)b * s.C * T + (long long)c * T + k) * P + p] = v;
        }
    }
}

// one thread per (b, group, tap, p): reduce over the group's channels
__global__ void dcn_col2im_coord_kernel(const float *__restrict__ gcol, const float *__restrict__ x,
                                        const float *__restrict__ offset, const float *__restrict__ mask,
                                        const c2m_dcn_shape s, const DcnGeom d, float *__restrict__ goff,
                                        float *__restrict__ gmask) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.dg * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), grp = (int)((e / ((long long)P * T)) % s.dg);
        const int b = (int)(e / ((long long)P * T * s.dg));
        const long long j = ((long long)b * s.dg + grp) * T + k;
        float h_im, w_im;
        float acc_h = 0.f, acc_w = 0.f, acc_m = 0.f;
        if (dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) {
            const float m = mask[j * P + p];
            const DcnCorners q(h_im, w_im, s.H, s.W, s.W, 1);
            const float hh = 1.f - q.lh, hw = 1.f - q.lw;
            for (int cl = 0; cl < cpg; ++cl) {
                const int c = grp * cpg + cl;
                const float gc = gcol[((long long)b * s.C * T + (long long)c * T + k) * P + p];
                const float *im = x + ((long long)b * s.C + c) * s.H * s.W;
                const float v1 = q.ok[0] ? im[q.o[0]] : 0.f, v2 = q.ok[1] ? im[q.o[1]] : 0.f;
                const float v3 = q.ok[2] ? im[q.o[2]] : 0.f, v4 = q.ok[3] ? im[q.o[3]] : 0.f;
                acc_m += gc * dcn_blend(q.w, v1, v2, v3, v4);
                acc_h += gc * m * (-hw * v1 - q.lw * v2 + hw * v3 + q.lw * v4);
                acc_w += gc * m * (-hh * v1 + hh * v2 - q.lh * v3 + q.lh * v4);
            }
        }
        goff[2 * j * P + p] = acc_h;
        goff[(2 * j + 1) * P + p] = acc_w;
        gmask[j * P + p] = acc_m;
    }
}

// one thread per (b, c, tap, p): scatter to the contributing corners
__global__ void dcn_col2im_kernel(const float *__restrict__ gcol, const float *__restrict__ offset,
                                  const float *__restrict__ mask, const c2m_dcn_shape s, const DcnGeom d,
                                  float *__restrict__ gx) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg;
    const long long n = (long long)s.B * s.C * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), c = (int)((e / ((long long)P * T)) % s.C);
        const int b = (int)(e / ((long long)P * T * s.C));
        const long long j = ((long long)b * s.dg + c / cpg) * T + k;
        float h_im, w_im;
        if (!dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) continue;
        const float tg = gcol[e] * mask[j * P + p];
        const DcnCorners q(h_im, w_im, s.H, s.W, s.W, 1);
        const float hh = 1.f - q.lh, hw = 1.f - q.lw;
        float *gim = gx + ((long long)b * s.C + c) * s.H * s.W;
        if (q.ok[0]) atomicAdd(gim + q.o[0], tg * hh * hw);
        if (q.ok[1]) atomicAdd(gim + q.o[1], tg * hh * q.lw);
        if (q.ok[2]) atomicAdd(gim + q.o[2], tg * q.lh * hw);
        if (q.ok[3]) atomicAdd(gim + q.o[3], tg * q.lh * q.lw);
    }
}

static inline int blocks_for(long long n) { long long b = (n + 255) / 256; return (int)(b > 132 * 16 ? 132 * 16 : b); }

}  // namespace c2m

using namespace c2m;

extern "C" int c2m_dcn_v2_im2col_f32(const float *x, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *columns, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && mask && columns, "dcn_v2_im2col: null pointer");
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_im2col_kernel<<<blocks_for((long long)shape->B * shape->C * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(x, offset, mask, *shape, d, columns);
    C2M_LAUNCH_CHECK("dcn_im2col_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_v2_col2im_coord_f32(const float *gcol, const float *x, const float *offset, const float *mask,
                                           const c2m_dcn_shape *shape, float *grad_offset, float *grad_mask,
                                           c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && x && offset && mask && grad_offset && grad_mask, "dcn_v2_col2im_coord: null pointer");
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_col2im_coord_kernel<<<blocks_for((long long)shape->B * shape->dg * d.T * d.Ho * d.Wo), 256, 0,
                              reinterpret_cast<cudaStream_t>(stream)>>>(gcol, x, offset, mask, *shape, d, grad_offset, grad_mask);
    C2M_LAUNCH_CHECK("dcn_col2im_coord_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_v2_col2im_f32(const float *gcol, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                                     float *grad_input, c2m_stream_t stream) {
    C2M_CHECK_ARG(gcol && offset && mask && grad_input, "dcn_v2_col2im: null pointer");
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_col2im_kernel<<<blocks_for((long long)shape->B * shape->C * d.T * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(gcol, offset, mask, *shape, d, grad_input);
    C2M_LAUNCH_CHECK("dcn_col2im_kernel");
    return C2M_OK;
}
