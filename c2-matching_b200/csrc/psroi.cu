// Deformable position-sensitive ROI pooling, forward and backward, fp32 and fp64 (`_ext.dcn_v2_psroi_pooling_forward`
// / `_backward`, DCNv2/src/dcn_v2.h:75-144, semantics of src/cuda/dcn_v2_psroi_pooling_cuda.cu:58-419).
//
// Output (n, c, ph, pw) averages the bilinear samples of bin (ph, pw) of ROI n in channel c.  The sampling geometry
// depends only on (ROI, bin, class), not on the channel, so a CTA owns (ROI, run of bins) x (class, run of channels):
// it writes the sample table of its bins once into shared memory — per sample the packed corner offset, the two
// fractional distances, or "skipped" — and then walks (channel, bin) pairs with the bin fastest, so that the stores of
// one channel's bins coalesce and a warp's gathers stay inside one or two channel planes.
//
// Sampling rule (local to this op; it is not DCN's): a sample outside [-0.5, W-0.5] x [-0.5, H-0.5] is dropped, a kept
// one is clamped to [0, W-1] x [0, H-1] and blends its floor / ceil corners, with no per-corner validity test.  The
// sample positions are computed in T with explicitly rounded multiplies and adds (no FMA contraction), in the
// reference's order, so the kernel takes the same skip / clamp branches as the plain-C oracle.
//
// Backward: grad_input is scattered with atomicAdd (summation order arbitrary).  grad_trans is reproducible bit for bit:
// each (ROI, channel, bin) writes its partial sum over samples to a caller-owned workspace, and a second kernel adds the
// partials of each (ROI, class, part cell) in a fixed order (bins ascending, then channels ascending).  With torch's
// deterministic algorithms on, grad_input comes instead from the ordered gather below (det_gather.cuh).
//
// Deliberate differences from the reference, which reads out of bounds in each case: C != output_dim, group_size != 1,
// a class count that does not divide output_dim and pooled_size / part_size / sample_per_part below 1 are rejected
// (C2M_ERR_INVALID); an ROI whose batch index, truncated toward zero, lies outside [0, B) pools to 0 with count 0 and
// receives no gradient.
#include "c2m_common.cuh"
#include "det_gather.cuh"

namespace c2m {

constexpr int PS_THREADS = 256;
constexpr int PS_MAX_SAMPLES = 2048;    // sample-table entries per CTA (fp64: 40 KB of shared memory)

// correctly rounded T arithmetic that the compiler may not fuse into an FMA
__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float rn_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rn_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double rn_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double rn_sub(double a, double b) { return __dsub_rn(a, b); }

struct PsroiLaunch {
    int bins_per_cta, tiles;      // bin runs per ROI
    int ch_per_cta, slices;       // channel runs per class
};

// Geometry of one ROI, in T.
template <typename T>
struct PsroiRoi {
    int b;                        // batch index, -1 when outside [0, B)
    T start_w, start_h, width, height, bin_w, bin_h, sub_w, sub_h;

    __device__ PsroiRoi(const T *roi, const c2m_psroi_shape &s) {
        const int bi = (int)roi[0];                                   // truncation toward zero
        b = bi >= 0 && bi < s.B && s.H > 0 && s.W > 0 ? bi : -1;
        const T scale = (T)s.spatial_scale;
        const T half = (T)0.5, one = (T)1;
        start_w = rn_sub(rn_mul((T)round(roi[1]), scale), half);
        start_h = rn_sub(rn_mul((T)round(roi[2]), scale), half);
        const T end_w = rn_sub(rn_mul(rn_add((T)round(roi[3]), one), scale), half);
        const T end_h = rn_sub(rn_mul(rn_add((T)round(roi[4]), one), scale), half);
        const T dw = rn_sub(end_w, start_w), dh = rn_sub(end_h, start_h);
        width = (double)dw > 0.1 ? dw : (T)0.1;                       // max(size, 0.1) with 0.1 a double
        height = (double)dh > 0.1 ? dh : (T)0.1;
        bin_w = width / (T)s.pooled_size;
        bin_h = height / (T)s.pooled_size;
        sub_w = bin_w / (T)s.sample_per_part;
        sub_h = bin_h / (T)s.sample_per_part;
    }
};

// part cell of bin coordinate p: floor(T(p) / P * part)
template <typename T>
__device__ __forceinline__ int psroi_part(int p, int P, int part) {
    return (int)floor(rn_mul((T)p / (T)P, (T)part));
}

// One sample of the bilinear rule.  code = (y0 * W + x0) << 2 | (x1 != x0) | (y1 != y0) << 1, or -1 when dropped;
// lx, ly = the distances from the floor corner.
template <typename T>
__device__ __forceinline__ void psroi_sample(T w, T h, int H, int W, int &code, T &lx, T &ly) {
    if ((double)w < -0.5 || (double)w > W - 0.5 || (double)h < -0.5 || (double)h > H - 0.5) {
        code = -1;
        lx = ly = (T)0;
        return;
    }
    w = (T)fmin(fmax((double)w, 0.), W - 1.);
    h = (T)fmin(fmax((double)h, 0.), H - 1.);
    const int x0 = (int)floor(w), x1 = (int)ceil(w), y0 = (int)floor(h), y1 = (int)ceil(h);
    lx = w - (T)x0;
    ly = h - (T)y0;
    code = ((y0 * W + x0) << 2) | (x1 != x0 ? 1 : 0) | (y1 != y0 ? 2 : 0);
}

// Position (w, h) of sample (ih, iw) of bin (ph, pw) of ROI n (geometry r) for class cls, translated by trans unless
// no_trans; psroi_sample turns it into corners.
template <typename T>
__device__ __forceinline__ void psroi_position(const PsroiRoi<T> &r, const T *trans, const c2m_psroi_shape &s, int n,
                                               int cls, int ph, int pw, int ih, int iw, T &w, T &h) {
    const int P = s.pooled_size, part = s.part_size;
    T tx = (T)0, ty = (T)0;
    if (!s.no_trans) {
        const int pcell = psroi_part<T>(ph, P, part) * part + psroi_part<T>(pw, P, part);
        const long long t0 = (((long long)n * s.num_classes + cls) * 2) * part * part + pcell;
        const T tstd = (T)s.trans_std;
        tx = rn_mul(trans[t0], tstd);
        ty = rn_mul(trans[t0 + (long long)part * part], tstd);
    }
    const T ws = rn_add(rn_add(rn_mul((T)pw, r.bin_w), r.start_w), rn_mul(tx, r.width));
    const T hs = rn_add(rn_add(rn_mul((T)ph, r.bin_h), r.start_h), rn_mul(ty, r.height));
    w = rn_add(ws, rn_mul((T)iw, r.sub_w));
    h = rn_add(hs, rn_mul((T)ih, r.sub_h));
}

// Shared-memory sample table of `nb` bins starting at bin0, S*S samples each: sample s = ih * S + iw of bin j at
// s * nb + j, so the threads of a warp, which walk consecutive bins, read consecutive words (no bank conflicts).  The
// ROI's translation for (class, part cell) is read from trans unless no_trans.
template <typename T>
struct PsroiTable {
    T *lx, *ly;
    int *code;

    __device__ PsroiTable(unsigned char *smem, int n) {
        lx = reinterpret_cast<T *>(smem);
        ly = lx + n;
        code = reinterpret_cast<int *>(ly + n);
    }

    __device__ void fill(const PsroiRoi<T> &r, const T *trans, const c2m_psroi_shape &s, int n, int cls, int bin0,
                         int nb) {
        const int P = s.pooled_size, S = s.sample_per_part, SS = S * S;
        for (int i = threadIdx.x; i < nb * SS; i += blockDim.x) {
            const int bin = bin0 + i % nb, ph = bin / P, pw = bin % P, ih = (i / nb) / S, iw = (i / nb) % S;
            if (r.b < 0) {
                code[i] = -1;
                lx[i] = ly[i] = (T)0;
                continue;
            }
            T w, h;
            psroi_position(r, trans, s, n, cls, ph, pw, ih, iw, w, h);
            psroi_sample(w, h, s.H, s.W, code[i], lx[i], ly[i]);
        }
    }
};

__device__ __forceinline__ void psroi_corners(int code, int W, int &o00, int &dx, int &dy) {
    o00 = code >> 2;
    dx = code & 1;
    dy = (code & 2) ? W : 0;
}

// blockIdx.x = ROI * tiles + bin run, blockIdx.y = class * slices + channel run
struct PsroiBlock {
    int n, bin0, nb, cls, c0, nc;
    __device__ PsroiBlock(const c2m_psroi_shape &s, const PsroiLaunch &L) {
        const int PP = s.pooled_size * s.pooled_size, cpc = s.output_dim / s.num_classes;
        n = blockIdx.x / L.tiles;
        bin0 = (blockIdx.x % L.tiles) * L.bins_per_cta;
        nb = min(L.bins_per_cta, PP - bin0);
        cls = blockIdx.y / L.slices;
        const int cl0 = (blockIdx.y % L.slices) * L.ch_per_cta;
        c0 = cls * cpc + cl0;
        nc = min(L.ch_per_cta, cpc - cl0);
    }
};

template <typename T>
__global__ void __launch_bounds__(PS_THREADS) psroi_fwd_kernel(const T *__restrict__ x, const T *__restrict__ bbox,
                                                               const T *__restrict__ trans, const c2m_psroi_shape s,
                                                               const PsroiLaunch L, T *__restrict__ out,
                                                               T *__restrict__ count) {
    extern __shared__ __align__(16) unsigned char smem[];
    const PsroiBlock blk(s, L);
    const int SS = s.sample_per_part * s.sample_per_part, PP = s.pooled_size * s.pooled_size;
    PsroiTable<T> tab(smem, blk.nb * SS);
    const PsroiRoi<T> roi(bbox + (long long)blk.n * 5, s);
    tab.fill(roi, trans, s, blk.n, blk.cls, blk.bin0, blk.nb);
    __syncthreads();

    const long long plane = (long long)s.H * s.W;
    for (int it = threadIdx.x; it < blk.nc * blk.nb; it += blockDim.x) {
        const int c = blk.c0 + it / blk.nb, j = it % blk.nb;
        const T *im = x + ((long long)(roi.b < 0 ? 0 : roi.b) * s.C + c) * plane;
        T sum = (T)0;
        int cnt = 0;
        for (int k = j; k < SS * blk.nb; k += blk.nb) {
            const int code = tab.code[k];
            if (code < 0) continue;
            int o, dx, dy;
            psroi_corners(code, s.W, o, dx, dy);
            const T lx = tab.lx[k], ly = tab.ly[k];
            sum += ((T)1 - lx) * ((T)1 - ly) * im[o] + ((T)1 - lx) * ly * im[o + dy] +
                   lx * ((T)1 - ly) * im[o + dx] + lx * ly * im[o + dx + dy];
            ++cnt;
        }
        const long long oi = ((long long)blk.n * s.output_dim + c) * PP + blk.bin0 + j;
        out[oi] = cnt == 0 ? (T)0 : sum / (T)cnt;
        count[oi] = (T)cnt;
    }
}

// grad_input += scatter; ws[(n, c, bin)] = this (channel, bin)'s unscaled trans-gradient partials (x, y) when trans is
// used.  The caller zero-fills grad_input.
template <typename T>
__global__ void __launch_bounds__(PS_THREADS) psroi_bwd_kernel(const T *__restrict__ gout, const T *__restrict__ x,
                                                               const T *__restrict__ bbox, const T *__restrict__ trans,
                                                               const T *__restrict__ top_count,
                                                               const c2m_psroi_shape s, const PsroiLaunch L,
                                                               T *__restrict__ gx, T *__restrict__ ws) {
    extern __shared__ __align__(16) unsigned char smem[];
    const PsroiBlock blk(s, L);
    const int SS = s.sample_per_part * s.sample_per_part, PP = s.pooled_size * s.pooled_size;
    PsroiTable<T> tab(smem, blk.nb * SS);
    const PsroiRoi<T> roi(bbox + (long long)blk.n * 5, s);
    tab.fill(roi, trans, s, blk.n, blk.cls, blk.bin0, blk.nb);
    __syncthreads();

    const long long plane = (long long)s.H * s.W;
    const T tstd = (T)s.trans_std;
    for (int it = threadIdx.x; it < blk.nc * blk.nb; it += blockDim.x) {
        const int c = blk.c0 + it / blk.nb, j = it % blk.nb;
        const long long oi = ((long long)blk.n * s.output_dim + c) * PP + blk.bin0 + j;
        const T cnt = top_count[oi];
        T acc_x = (T)0, acc_y = (T)0;
        if (roi.b >= 0 && cnt > (T)0) {
            const T diff = gout[oi] / cnt;
            const long long base = ((long long)roi.b * s.C + c) * plane;
            const T *im = x + base;
            T *gim = gx + base;
            for (int k = j; k < SS * blk.nb; k += blk.nb) {
                const int code = tab.code[k];
                if (code < 0) continue;
                int o, dx, dy;
                psroi_corners(code, s.W, o, dx, dy);
                const T lx = tab.lx[k], ly = tab.ly[k], hx = (T)1 - lx, hy = (T)1 - ly;
                // a corner that coincides with the floor corner has weight 0: only distinct corners are written
                atomicAdd(gim + o, hx * hy * diff);
                if (dy) atomicAdd(gim + o + dy, hx * ly * diff);
                if (dx) atomicAdd(gim + o + dx, lx * hy * diff);
                if (dx && dy) atomicAdd(gim + o + dx + dy, lx * ly * diff);
                if (!s.no_trans) {
                    const T u00 = im[o], u01 = im[o + dy], u10 = im[o + dx], u11 = im[o + dx + dy];
                    acc_x += u11 * ly + u10 * hy - u01 * ly - u00 * hy;
                    acc_y += u11 * lx + u01 * hx - u10 * lx - u00 * hx;
                }
            }
            acc_x = acc_x * tstd * diff * roi.width;
            acc_y = acc_y * tstd * diff * roi.height;
        }
        if (!s.no_trans) {
            ws[2 * oi] = acc_x;
            ws[2 * oi + 1] = acc_y;
        }
    }
}

// grad_trans[n, cls, {x, y}, part_h, part_w] = sum over the bins of that part cell (ascending), then the class's
// channels (ascending), of ws.  One thread per (n, cls, part cell); every element is written.
template <typename T>
__global__ void psroi_trans_grad_kernel(const T *__restrict__ ws, const c2m_psroi_shape s, T *__restrict__ gtrans) {
    const int part = s.part_size, P = s.pooled_size, PP = P * P, K = s.num_classes, cpc = s.output_dim / K;
    const long long total = (long long)s.R * K * part * part;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const int pw_ = (int)(e % part), ph_ = (int)((e / part) % part), cls = (int)((e / (part * part)) % K);
        const long long n = e / ((long long)part * part * K);
        T gxs = (T)0, gys = (T)0;
        for (int ph = 0; ph < P; ++ph) {
            if (psroi_part<T>(ph, P, part) != ph_) continue;
            for (int pw = 0; pw < P; ++pw) {
                if (psroi_part<T>(pw, P, part) != pw_) continue;
                for (int c = cls * cpc; c < (cls + 1) * cpc; ++c) {
                    const long long oi = (n * s.output_dim + c) * PP + ph * P + pw;
                    gxs += ws[2 * oi];
                    gys += ws[2 * oi + 1];
                }
            }
        }
        const long long t0 = ((n * K + cls) * 2) * part * part + ph_ * part + pw_;
        gtrans[t0] = gxs;
        gtrans[t0 + part * part] = gys;
    }
}

// ---- ordered grad_input (det_gather.cuh).  Plane q = (image b, class cls) = b * K + cls; its entries are
// id = ((n * PP + bin) * SS + sample) * 4 + corner with corners floor, +dy, +dx, +dx+dy, so ascending id is ascending
// ROI, bin (row-major), sample (row-major), corner.  Entries of ROIs of other images, dropped samples and corners that
// coincide with the floor corner get the "no pixel" key.

// one thread per (plane of the pass, ROI, bin, sample)
template <typename T>
__global__ void psroi_grad_emit_kernel(const T *__restrict__ bbox, const T *__restrict__ trans,
                                       const c2m_psroi_shape s, int q0, int np, uint32_t *__restrict__ keys,
                                       uint32_t *__restrict__ ids) {
    const int P = s.pooled_size, PP = P * P, S = s.sample_per_part, SS = S * S, HW = s.H * s.W;
    const long long per = (long long)s.R * PP * SS, total = np * per;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long local = e % per;
        const int si = (int)(local % SS), bin = (int)((local / SS) % PP), n = (int)(local / ((long long)SS * PP));
        const int ql = (int)(e / per), q = q0 + ql, b = q / s.num_classes, cls = q % s.num_classes;
        const uint32_t key0 = (uint32_t)ql * (uint32_t)(HW + 1);
        uint32_t key[4] = {key0 + HW, key0 + HW, key0 + HW, key0 + HW};
        const PsroiRoi<T> roi(bbox + (long long)n * 5, s);
        if (roi.b == b) {
            int code;
            T lx, ly;
            T w, h;
            psroi_position(roi, trans, s, n, cls, bin / P, bin % P, si / S, si % S, w, h);
            psroi_sample(w, h, s.H, s.W, code, lx, ly);
            if (code >= 0) {
                int o, dx, dy;
                psroi_corners(code, s.W, o, dx, dy);
                key[0] = key0 + (uint32_t)o;
                if (dy) key[1] = key0 + (uint32_t)(o + dy);
                if (dx) key[2] = key0 + (uint32_t)(o + dx);
                if (dx && dy) key[3] = key0 + (uint32_t)(o + dx + dy);
            }
        }
        const uint32_t id0 = (uint32_t)local * 4u;
        const long long base = ql * per * 4 + id0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            keys[base + c] = key[c];
            ids[base + c] = id0 + c;
        }
    }
}

constexpr int PS_GATHER_CH = 4;    // channels of a class one gather thread accumulates

// one thread per (plane of the pass, run of PS_GATHER_CH channels of its class, input pixel): walks the pixel's sorted
// entries, recomputes each sample once and adds (hx * hy) * (out_grad / count) and so on, as psroi_bwd_kernel, to
// every channel of the run whose count is positive, with correctly rounded adds from +0.  Writes every element.
template <typename T>
__global__ void psroi_grad_gather_kernel(const T *__restrict__ gout, const T *__restrict__ bbox,
                                         const T *__restrict__ trans, const T *__restrict__ top_count,
                                         const c2m_psroi_shape s, int q0, int np, const uint32_t *__restrict__ seg,
                                         const uint32_t *__restrict__ ids, T *__restrict__ gx) {
    const int P = s.pooled_size, PP = P * P, S = s.sample_per_part, SS = S * S, HW = s.H * s.W;
    const int cpc = s.output_dim / s.num_classes, runs = ceil_div(cpc, PS_GATHER_CH);
    const long long total = (long long)np * runs * HW;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const int pix = (int)(e % HW), r = (int)((e / HW) % runs), ql = (int)(e / ((long long)HW * runs));
        const int q = q0 + ql, b = q / s.num_classes, cls = q % s.num_classes;
        const int c0 = cls * cpc + r * PS_GATHER_CH, nc = min(PS_GATHER_CH, cpc - r * PS_GATHER_CH);
        T acc[PS_GATHER_CH];
#pragma unroll
        for (int i = 0; i < PS_GATHER_CH; ++i) acc[i] = (T)0;
        const uint32_t key = (uint32_t)ql * (uint32_t)(HW + 1) + (uint32_t)pix;
        for (uint32_t it = seg[key], end = seg[key + 1]; it < end; ++it) {
            const uint32_t id = ids[it], t = id >> 2, corner = id & 3u;
            const int si = (int)(t % (uint32_t)SS), bin = (int)((t / (uint32_t)SS) % (uint32_t)PP);
            const int n = (int)(t / ((uint32_t)SS * (uint32_t)PP));
            const PsroiRoi<T> roi(bbox + (long long)n * 5, s);
            int code;
            T lx, ly;
            T w, h;
            psroi_position(roi, trans, s, n, cls, bin / P, bin % P, si / S, si % S, w, h);
            psroi_sample(w, h, s.H, s.W, code, lx, ly);
            const T hx = (T)1 - lx, hy = (T)1 - ly;
            const T wgt = corner == 0 ? hx * hy : corner == 1 ? hx * ly : corner == 2 ? lx * hy : lx * ly;
            const long long oi0 = ((long long)n * s.output_dim + c0) * PP + bin;
#pragma unroll
            for (int i = 0; i < PS_GATHER_CH; ++i) {
                if (i >= nc) continue;
                const T cnt = top_count[oi0 + (long long)i * PP];
                if (cnt > (T)0) acc[i] = rn_add(acc[i], wgt * (gout[oi0 + (long long)i * PP] / cnt));
            }
        }
        T *out = gx + ((long long)b * s.C + c0) * HW + pix;
#pragma unroll
        for (int i = 0; i < PS_GATHER_CH; ++i)
            if (i < nc) out[(long long)i * HW] = acc[i];
    }
}

static int psroi_check(const c2m_psroi_shape *s, const char *what) {
    C2M_CHECK_ARG(s, "%s: null shape", what);
    C2M_CHECK_ARG(s->B >= 0 && s->C >= 0 && s->H >= 0 && s->W >= 0 && s->R >= 0 && s->output_dim >= 0,
                  "%s: negative size", what);
    C2M_CHECK_ARG(s->C == s->output_dim, "%s: input channels and output channels must equal (%d vs %d)", what, s->C,
                  s->output_dim);
    C2M_CHECK_ARG(s->group_size == 1, "%s: group_size must be 1 (got %d): with C == output_dim any larger group reads "
                  "channels beyond C", what, s->group_size);
    C2M_CHECK_ARG(s->pooled_size >= 1 && s->part_size >= 1 && s->sample_per_part >= 1,
                  "%s: pooled_size, part_size and sample_per_part must be >= 1 (got %d, %d, %d)", what, s->pooled_size,
                  s->part_size, s->sample_per_part);
    C2M_CHECK_ARG(s->sample_per_part * s->sample_per_part <= PS_MAX_SAMPLES, "%s: sample_per_part above 45 is not "
                  "supported (got %d)", what, s->sample_per_part);
    C2M_CHECK_ARG(s->no_trans || s->num_classes >= 1, "%s: trans must have 2 * K channels with K >= 1", what);
    C2M_CHECK_ARG(s->no_trans || s->output_dim % s->num_classes == 0,
                  "%s: output_dim (%d) must be a multiple of the number of trans classes (%d)", what, s->output_dim,
                  s->num_classes);
    C2M_CHECK_ARG((long long)s->H * s->W < (1ll << 29), "%s: feature map of %d x %d pixels is too large", what, s->H,
                  s->W);
    return C2M_OK;
}

// Bin runs keep a CTA's table within PS_MAX_SAMPLES; channel runs of 8..64 are halved while the grid has fewer than
// four CTAs per SM of an H100, so small ROI counts still fill the device.
static PsroiLaunch psroi_launch(const c2m_psroi_shape &s) {
    PsroiLaunch L;
    const int PP = s.pooled_size * s.pooled_size, SS = s.sample_per_part * s.sample_per_part;
    L.bins_per_cta = PP * SS <= PS_MAX_SAMPLES ? PP : PS_MAX_SAMPLES / SS;
    L.tiles = ceil_div(PP, L.bins_per_cta);
    const int K = s.no_trans ? 1 : s.num_classes, cpc = s.output_dim / K;
    int cs = cpc < 64 ? cpc : 64;
    while (cs > 8 && (long long)s.R * L.tiles * K * ceil_div(cpc, cs) < 4 * 132) cs = (cs + 1) / 2;
    L.slices = ceil_div(cpc, cs);
    L.ch_per_cta = ceil_div(cpc, L.slices);
    return L;
}

template <typename T>
static size_t psroi_smem(const c2m_psroi_shape &s, const PsroiLaunch &L) {
    return (size_t)L.bins_per_cta * s.sample_per_part * s.sample_per_part * (2 * sizeof(T) + sizeof(int));
}

static c2m_psroi_shape psroi_effective(const c2m_psroi_shape &s) {
    c2m_psroi_shape e = s;
    if (e.no_trans) e.num_classes = 1;   // one class spanning every channel
    return e;
}

template <typename T>
static int psroi_forward(const T *x, const T *bbox, const T *trans, const c2m_psroi_shape *shape, T *out, T *count,
                         c2m_stream_t stream) {
    if (int rc = psroi_check(shape, "psroi_pooling_forward")) return rc;
    const c2m_psroi_shape s = psroi_effective(*shape);
    if (s.R == 0 || s.output_dim == 0) return C2M_OK;
    C2M_CHECK_ARG((x || (long long)s.B * s.C * s.H * s.W == 0) && bbox && out && count && (s.no_trans || trans),
                  "psroi_pooling_forward: null pointer");
    const PsroiLaunch L = psroi_launch(s);
    C2M_CHECK_ARG(s.num_classes * L.slices <= 65535, "psroi_pooling_forward: too many channels (%d)", s.output_dim);
    const dim3 grid((unsigned)(s.R * L.tiles), (unsigned)(s.num_classes * L.slices));
    psroi_fwd_kernel<T><<<grid, PS_THREADS, psroi_smem<T>(s, L), reinterpret_cast<cudaStream_t>(stream)>>>(
        x, bbox, trans, s, L, out, count);
    C2M_LAUNCH_CHECK("psroi_fwd_kernel");
    return C2M_OK;
}

template <typename T>
static int psroi_backward(const T *gout, const T *x, const T *bbox, const T *trans, const T *top_count,
                          const c2m_psroi_shape *shape, T *grad_input, T *grad_trans, void *ws, size_t ws_bytes,
                          c2m_stream_t stream) {
    if (int rc = psroi_check(shape, "psroi_pooling_backward")) return rc;
    const c2m_psroi_shape s = psroi_effective(*shape);
    if (s.R == 0 || s.output_dim == 0 || (long long)s.B * s.H * s.W == 0) return C2M_OK;
    C2M_CHECK_ARG(gout && x && bbox && top_count && grad_input && (s.no_trans || (trans && grad_trans)),
                  "psroi_pooling_backward: null pointer");
    const size_t need = c2m_psroi_pooling_workspace_bytes(shape, (int)sizeof(T));
    C2M_CHECK_ARG(ws_bytes >= need && (need == 0 || ws), "psroi_pooling_backward: workspace of %zu bytes given, %zu "
                  "needed", ws_bytes, need);
    const PsroiLaunch L = psroi_launch(s);
    C2M_CHECK_ARG(s.num_classes * L.slices <= 65535, "psroi_pooling_backward: too many channels (%d)", s.output_dim);
    const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)(s.R * L.tiles), (unsigned)(s.num_classes * L.slices));
    psroi_bwd_kernel<T><<<grid, PS_THREADS, psroi_smem<T>(s, L), st>>>(gout, x, bbox, trans, top_count, s, L,
                                                                        grad_input, static_cast<T *>(ws));
    C2M_LAUNCH_CHECK("psroi_bwd_kernel");
    if (!s.no_trans) {
        const long long cells = (long long)s.R * s.num_classes * s.part_size * s.part_size;
        psroi_trans_grad_kernel<T><<<grid_blocks(cells), 256, 0, st>>>(static_cast<const T *>(ws), s, grad_trans);
        C2M_LAUNCH_CHECK("psroi_trans_grad_kernel");
    }
    return C2M_OK;
}

template <typename T>
static int psroi_grad_input_det(const T *gout, const T *bbox, const T *trans, const T *top_count,
                                const c2m_psroi_shape *shape, T *grad_input, void *ws, size_t ws_bytes,
                                c2m_stream_t stream) {
    const char *who = "psroi_pooling_grad_input_det";
    if (int rc = psroi_check(shape, who)) return rc;
    const c2m_psroi_shape s = psroi_effective(*shape);
    const long long nx = (long long)s.B * s.C * s.H * s.W;
    if (nx == 0) return C2M_OK;
    C2M_CHECK_ARG(grad_input, "%s: null pointer", who);
    const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (s.R == 0) {                                       // no ROI: every element is +0
        C2M_CUDA(cudaMemsetAsync(grad_input, 0, (size_t)nx * sizeof(T), st));
        return C2M_OK;
    }
    C2M_CHECK_ARG(gout && bbox && top_count && (s.no_trans || trans) && ws, "%s: null pointer", who);
    const long long E = 4ll * s.R * s.pooled_size * s.pooled_size * s.sample_per_part * s.sample_per_part;
    const long long K = (long long)s.H * s.W + 1;
    if (!det_plane_fits(E, K, who)) return C2M_ERR_INVALID;
    const int runs = ceil_div(s.output_dim / s.num_classes, PS_GATHER_CH);
    auto emit = [&](int q0, int n, uint32_t *keys, uint32_t *ids) -> int {
        psroi_grad_emit_kernel<T><<<grid_blocks(n * E / 4), 256, 0, st>>>(bbox, trans, s, q0, n, keys, ids);
        C2M_LAUNCH_CHECK("psroi_grad_emit_kernel");
        return C2M_OK;
    };
    auto gather = [&](int q0, int n, const uint32_t *seg, const uint32_t *ids) -> int {
        psroi_grad_gather_kernel<T><<<grid_blocks((long long)n * runs * s.H * s.W), 256, 0, st>>>(
            gout, bbox, trans, top_count, s, q0, n, seg, ids, grad_input);
        C2M_LAUNCH_CHECK("psroi_grad_gather_kernel");
        return C2M_OK;
    };
    return det_passes(ws, ws_bytes, (long long)s.B * s.num_classes, E, K, who, st, emit, gather);
}

}  // namespace c2m

using namespace c2m;

extern "C" size_t c2m_psroi_pooling_workspace_bytes(const c2m_psroi_shape *shape, int elem_bytes) {
    if (!shape || shape->no_trans || shape->R <= 0 || shape->output_dim <= 0 || shape->pooled_size <= 0) return 0;
    return (size_t)shape->R * shape->output_dim * shape->pooled_size * shape->pooled_size * 2 * (size_t)elem_bytes;
}

extern "C" int c2m_psroi_pooling_forward_f32(const float *input, const float *bbox, const float *trans,
                                             const c2m_psroi_shape *shape, float *out, float *count,
                                             c2m_stream_t stream) {
    return psroi_forward(input, bbox, trans, shape, out, count, stream);
}

extern "C" int c2m_psroi_pooling_forward_f64(const double *input, const double *bbox, const double *trans,
                                             const c2m_psroi_shape *shape, double *out, double *count,
                                             c2m_stream_t stream) {
    return psroi_forward(input, bbox, trans, shape, out, count, stream);
}

extern "C" int c2m_psroi_pooling_backward_f32(const float *out_grad, const float *input, const float *bbox,
                                              const float *trans, const float *top_count, const c2m_psroi_shape *shape,
                                              float *grad_input, float *grad_trans, void *ws, size_t ws_bytes,
                                              c2m_stream_t stream) {
    return psroi_backward(out_grad, input, bbox, trans, top_count, shape, grad_input, grad_trans, ws, ws_bytes, stream);
}

extern "C" int c2m_psroi_pooling_backward_f64(const double *out_grad, const double *input, const double *bbox,
                                              const double *trans, const double *top_count,
                                              const c2m_psroi_shape *shape, double *grad_input, double *grad_trans,
                                              void *ws, size_t ws_bytes, c2m_stream_t stream) {
    return psroi_backward(out_grad, input, bbox, trans, top_count, shape, grad_input, grad_trans, ws, ws_bytes, stream);
}

extern "C" size_t c2m_psroi_grad_input_det_workspace_bytes(const c2m_psroi_shape *shape, int planes) {
    const char *who = "psroi_grad_input_det_workspace_bytes";
    if (psroi_check(shape, who)) return 0;
    const c2m_psroi_shape s = psroi_effective(*shape);
    const long long E = 4ll * s.R * s.pooled_size * s.pooled_size * s.sample_per_part * s.sample_per_part;
    const long long K = (long long)s.H * s.W + 1;
    if (!det_plane_fits(E, K, who)) return 0;
    return det_workspace_bytes(planes, (long long)s.B * s.num_classes, E, K, who);
}

extern "C" int c2m_psroi_pooling_grad_input_det_f32(const float *out_grad, const float *bbox, const float *trans,
                                                    const float *top_count, const c2m_psroi_shape *shape,
                                                    float *grad_input, void *ws, size_t ws_bytes,
                                                    c2m_stream_t stream) {
    return psroi_grad_input_det(out_grad, bbox, trans, top_count, shape, grad_input, ws, ws_bytes, stream);
}

extern "C" int c2m_psroi_pooling_grad_input_det_f64(const double *out_grad, const double *bbox, const double *trans,
                                                    const double *top_count, const c2m_psroi_shape *shape,
                                                    double *grad_input, void *ws, size_t ws_bytes,
                                                    c2m_stream_t stream) {
    return psroi_grad_input_det(out_grad, bbox, trans, top_count, shape, grad_input, ws, ws_bytes, stream);
}
