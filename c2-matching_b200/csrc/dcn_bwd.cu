// DCNv2 backward building blocks (SURVEY.md §8f N4; completes the `_ext` ABI:
// `_ext.dcn_v2_backward`, DCNv2/src/dcn_v2.h:41-72, dcn_v2_cuda.cu:206-335).
//
// Training is not on the restoration-forward hot path, so this keeps the reference's
// decomposition — column-gradient GEMM, coordinate/mask gradient, input-gradient scatter, column
// matrix for the weight gradient — with the two dense GEMMs left to the caller (torch.matmul) and
// the three deformable pieces written here:
//   c2m_deform_conv_im2col_*        columns[b, c*T+k, p] = mask * bilinear(x)       (:125-195)
//   c2m_deform_conv_col2im_coord_*  grad_offset / grad_mask from gcol                (:256-327, 83-123)
//   c2m_deform_conv_col2im_*        grad_input += scatter of gcol * mask             (:197-254, 56-80)
// Unlike the reference, batch is a grid dimension (no host loop), grad_input scatter touches only
// the (<= 4) contributing corners instead of a 5x5 window, and launch errors are returned.
// Sampling points, corners and the shape check are the forward's (dcn_sampling.cuh); a corner
// outside the image is skipped here, where the forward loads element 0 with weight 0.
//
// The kernels are templated on the scalar type and serve `_ext` (fp32, with a mask) and `deform_conv_cuda`
// (mmsr/models/archs/dcn): a null mask is a modulation of 1 and then no grad_mask is written.  The reference's DCNv1
// kernels (deformable_im2col / col2im / col2im_coord, dcn/src/deform_conv_cuda_kernel.cu:116-434) are these formulas
// with m = 1, and their 5x5-window scatter reaches the same <= 4 corners.  Conv groups enter only the two GEMMs.
#include "dcn_sampling.cuh"
#include "det_gather.cuh"

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

// ---- ordered input gradient (det_gather.cuh).  Plane q = (image b, deformable group g) = b * dg + g; its entries are
// id = (k * P + p) * 4 + corner (corners in DcnCorners order), so ascending id is ascending tap, output pixel, corner.

__device__ __forceinline__ float dcn_add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double dcn_add_rn(double a, double b) { return __dadd_rn(a, b); }

// one thread per (plane of the pass, tap, p): the four entries of the sampling point
template <typename scalar_t>
__global__ void dcn_col2im_emit_kernel(const scalar_t *__restrict__ offset, const c2m_dcn_shape s, const DcnGeom d,
                                       int q0, int np, uint32_t *__restrict__ keys, uint32_t *__restrict__ ids) {
    const int T = d.T, P = d.Ho * d.Wo, HW = s.H * s.W;
    const long long n = (long long)np * T * P;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(e % P), k = (int)((e / P) % T), ql = (int)(e / ((long long)P * T));
        const long long j = (long long)(q0 + ql) * T + k;
        const uint32_t key0 = (uint32_t)ql * (uint32_t)(HW + 1), id0 = (uint32_t)(k * P + p) * 4u;
        uint32_t key[4] = {key0 + HW, key0 + HW, key0 + HW, key0 + HW};
        scalar_t h_im, w_im;
        if (dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im)) {
            const DcnCorners<scalar_t> q(h_im, w_im, s.H, s.W, s.W, 1);
#pragma unroll
            for (int c = 0; c < 4; ++c)
                if (q.ok[c]) key[c] = key0 + (uint32_t)q.o[c];
        }
        const long long base = (long long)ql * T * P * 4 + id0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            keys[base + c] = key[c];
            ids[base + c] = id0 + c;
        }
    }
}

constexpr int DCN_GATHER_CH = 4;   // channels of a deformable group one gather thread accumulates

// one thread per (plane of the pass, run of DCN_GATHER_CH channels of its group, input pixel): walks the pixel's
// sorted entries, recomputes each one's sampling point once and adds its contribution to every channel of the run,
// ((gcol * m) * hh) * hw and so on as in dcn_col2im_kernel, with correctly rounded adds from +0.  Writes every element.
template <typename scalar_t>
__global__ void dcn_col2im_gather_kernel(const scalar_t *__restrict__ gcol, const scalar_t *__restrict__ offset,
                                         const scalar_t *__restrict__ mask, const c2m_dcn_shape s, const DcnGeom d,
                                         int q0, int np, const uint32_t *__restrict__ seg,
                                         const uint32_t *__restrict__ ids, scalar_t *__restrict__ gx) {
    const int T = d.T, P = d.Ho * d.Wo, cpg = d.cpg, HW = s.H * s.W;
    const int runs = ceil_div(cpg, DCN_GATHER_CH);
    const long long n = (long long)np * runs * HW;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int pix = (int)(e % HW), r = (int)((e / HW) % runs), ql = (int)(e / ((long long)HW * runs));
        const int q = q0 + ql, b = q / s.dg, c0 = (q % s.dg) * cpg + r * DCN_GATHER_CH;
        const int nc = min(DCN_GATHER_CH, cpg - r * DCN_GATHER_CH);
        scalar_t acc[DCN_GATHER_CH];
#pragma unroll
        for (int i = 0; i < DCN_GATHER_CH; ++i) acc[i] = (scalar_t)0;
        const uint32_t key = (uint32_t)ql * (uint32_t)(HW + 1) + (uint32_t)pix;
        for (uint32_t it = seg[key], end = seg[key + 1]; it < end; ++it) {
            const uint32_t id = ids[it], kp = id >> 2, corner = id & 3u;
            const int k = (int)(kp / (uint32_t)P), p = (int)(kp % (uint32_t)P);
            const long long j = (long long)q * T + k;
            scalar_t h_im, w_im;
            dcn_sample_point(s, d.Wo, k, p, offset[2 * j * P + p], offset[(2 * j + 1) * P + p], h_im, w_im);
            const DcnCorners<scalar_t> cq(h_im, w_im, s.H, s.W, s.W, 1);
            const scalar_t wa = corner < 2 ? (scalar_t)1 - cq.lh : cq.lh;
            const scalar_t wb = (corner & 1u) ? cq.lw : (scalar_t)1 - cq.lw;
            const scalar_t m = mask ? mask[j * P + p] : (scalar_t)1;
            const scalar_t *gc = gcol + (((long long)b * s.C + c0) * T + k) * P + p;
#pragma unroll
            for (int i = 0; i < DCN_GATHER_CH; ++i)
                if (i < nc) acc[i] = dcn_add_rn(acc[i], gc[(long long)i * T * P] * m * wa * wb);
        }
        scalar_t *out = gx + ((long long)b * s.C + c0) * HW + pix;
#pragma unroll
        for (int i = 0; i < DCN_GATHER_CH; ++i)
            if (i < nc) out[(long long)i * HW] = acc[i];
    }
}

template <typename scalar_t>
static int col2im_det(const scalar_t *gcol, const scalar_t *offset, const scalar_t *mask, const c2m_dcn_shape *shape,
                      scalar_t *grad_input, void *ws, size_t ws_bytes, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn ordered col2im", d)) return rc;
    const long long E = 4ll * d.T * d.Ho * d.Wo, K = (long long)shape->H * shape->W + 1;
    if (!det_plane_fits(E, K, "dcn ordered col2im")) return C2M_ERR_INVALID;
    const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int runs = ceil_div(d.cpg, DCN_GATHER_CH);
    auto emit = [&](int q0, int n, uint32_t *keys, uint32_t *ids) -> int {
        dcn_col2im_emit_kernel<<<grid_blocks((long long)n * d.T * d.Ho * d.Wo), 256, 0, st>>>(offset, *shape, d, q0, n,
                                                                                             keys, ids);
        C2M_LAUNCH_CHECK("dcn_col2im_emit_kernel");
        return C2M_OK;
    };
    auto gather = [&](int q0, int n, const uint32_t *seg, const uint32_t *ids) -> int {
        dcn_col2im_gather_kernel<<<grid_blocks((long long)n * runs * shape->H * shape->W), 256, 0, st>>>(
            gcol, offset, mask, *shape, d, q0, n, seg, ids, grad_input);
        C2M_LAUNCH_CHECK("dcn_col2im_gather_kernel");
        return C2M_OK;
    };
    return det_passes(ws, ws_bytes, (long long)shape->B * shape->dg, E, K, "dcn ordered col2im", st, emit, gather);
}

template <typename scalar_t>
static int im2col(const scalar_t *x, const scalar_t *offset, const scalar_t *mask, const c2m_dcn_shape *shape,
                  scalar_t *columns, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_im2col_kernel<<<grid_blocks((long long)shape->B * shape->C * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(x, offset, mask, *shape, d, columns);
    C2M_LAUNCH_CHECK("dcn_im2col_kernel");
    return C2M_OK;
}

template <typename scalar_t>
static int col2im_coord(const scalar_t *gcol, const scalar_t *x, const scalar_t *offset, const scalar_t *mask,
                        const c2m_dcn_shape *shape, scalar_t *grad_offset, scalar_t *grad_mask, c2m_stream_t stream) {
    DcnGeom d;
    if (int rc = dcn_geometry(shape, "dcn backward", d)) return rc;
    dcn_col2im_coord_kernel<<<grid_blocks((long long)shape->B * shape->dg * d.T * d.Ho * d.Wo), 256, 0,
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
    dcn_col2im_kernel<<<grid_blocks((long long)shape->B * shape->C * d.T * d.Ho * d.Wo), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(gcol, offset, mask, *shape, d, grad_input);
    C2M_LAUNCH_CHECK("dcn_col2im_kernel");
    return C2M_OK;
}

}  // namespace c2m

using namespace c2m;

// mask may be NULL (DCNv1), and grad_mask is NULL exactly when mask is
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

// ordered input gradient: grad_input written (not accumulated), in the order of col2im_det
extern "C" size_t c2m_dcn_col2im_det_workspace_bytes(const c2m_dcn_shape *shape, int planes) {
    DcnGeom d;
    if (dcn_geometry(shape, "dcn_col2im_det_workspace_bytes", d)) return 0;
    const long long E = 4ll * d.T * d.Ho * d.Wo, K = (long long)shape->H * shape->W + 1;
    if (!det_plane_fits(E, K, "dcn_col2im_det_workspace_bytes")) return 0;
    return det_workspace_bytes(planes, (long long)shape->B * shape->dg, E, K, "dcn_col2im_det_workspace_bytes");
}

#define C2M_DEFORM_CONV_COL2IM_DET(T, SFX)                                                                          \
    extern "C" int c2m_deform_conv_col2im_det_##SFX(const T *gcol, const T *offset, const T *mask,                  \
                                                    const c2m_dcn_shape *shape, T *grad_input, void *ws,            \
                                                    size_t ws_bytes, c2m_stream_t stream) {                         \
        C2M_CHECK_ARG(gcol && offset && grad_input, "deform_conv_col2im_det: null pointer");                        \
        return col2im_det(gcol, offset, mask, shape, grad_input, ws, ws_bytes, stream);                             \
    }

C2M_DEFORM_CONV_COL2IM_DET(float, f32)
C2M_DEFORM_CONV_COL2IM_DET(double, f64)
