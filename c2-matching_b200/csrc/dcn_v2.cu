// Fused modulated deformable convolution v2 forward (fp32) for sm_90a.
//
// Replaces `_ext.dcn_v2_forward` (mmsr/models/archs/DCNv2/src/cuda/dcn_v2_cuda.cu:42-172): the
// reference writes the whole im2col matrix `columns[B, C*kh*kw, Ho*Wo]` to HBM (0.94 GB per image
// for the 64-ch 640x640 layer), reads it back in a batched SGEMM, broadcasts the bias with a
// second GEMM and does 6 cudaMalloc/Free per call.  Here one kernel does
//   sampling coordinates -> bilinear gather -> column tile in SHARED memory -> contraction with
//   the (smem-staged) weights -> bias (+ LeakyReLU) -> store,
// and the fused entry also absorbs DCN_sep_pre_multi_offset's prologue (dcn_v2.py:233-250:
// pre-offset add with the (x,y)->(y,x) reorder, sigmoid of the mask, no host sync) and can rebuild
// the pre-offsets from the index map on the fly (corres_generation_arch.py:29-46,70-104).
//
// The sampling rule, shape check and index-map decode are the ones in dcn_sampling.cuh, shared with
// the backward kernels (dcn_bwd.cu) and offsets.cu.
//
// CTA = 256 threads = 64 output pixels x (16*NO) output channels; thread (tx,ty) owns pixels
// 4tx..4tx+3 and channels ty+16i.  K is walked one deformable group / channel block at a time:
// the sampling table (4 corner offsets + 4 weights + mask per (tap, pixel)) is computed once
// and shared by all channels of the group.  A corner outside the image is stored as element 0
// with weight 0, so the gather loads unconditionally.
#include "dcn_sampling.cuh"

namespace c2m {

namespace {
constexpr int TP = 64;        // pixels per CTA
constexpr int KSUB = 32;      // K rows per weight sub-slice
constexpr int MAXT = 9;       // taps per pass
constexpr int MAXCB = 32;     // channels per pass

struct DcnArgs {
    const float *x, *offset, *mask, *om, *pre, *weight, *bias;
    const long long *idx;
    float *out;
    c2m_dcn_shape s;
    DcnGeom g;
    int gh, gw, ref_gw, pre_scale;
    float slope;
    int CB;                   // channels per pass (<= cpg, <= MAXCB)
};

struct Samp {
    int o[4];
    float w[4];
    float m;
};
}  // namespace

template <int NO>
__global__ void __launch_bounds__(256) dcn_fwd_kernel(const DcnArgs a) {
    extern __shared__ __align__(16) uint8_t dsm[];
    const c2m_dcn_shape &s = a.s;
    const int T = a.g.T, cpg = a.g.cpg, CB = a.CB;
    const int P = a.g.Ho * a.g.Wo;
    const int NOUT = 16 * NO;

    Samp *samp = reinterpret_cast<Samp *>(dsm);                               // [MAXT][TP]
    float *col = reinterpret_cast<float *>(dsm + sizeof(Samp) * MAXT * TP);   // [CB*MAXT][TP]
    float *Ws = col + (size_t)CB * MAXT * TP;                                 // [KSUB][NOUT]

    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int b = blockIdx.y, p0 = blockIdx.x * TP, o0 = blockIdx.z * NOUT;
    const float *xb = a.x + (long long)b * s.xs_b;

    float acc[NO][4];
#pragma unroll
    for (int i = 0; i < NO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int g = 0; g < s.dg; ++g) {
        for (int t0 = 0; t0 < T; t0 += MAXT) {
            const int TB = min(MAXT, T - t0);
            __syncthreads();
            // ---- sampling table for (tap, pixel), shared by the group's channels
            for (int e = t; e < TB * TP; e += 256) {
                const int tl = e / TP, pl = e % TP, tap = t0 + tl, p = p0 + pl;
                Samp sp = {};
                if (p < P) {
                    const int j = g * T + tap;
                    float off_h, off_w, m;
                    if (a.om) {
                        const float *omb = a.om + (long long)b * 3 * s.dg * T * P;
                        off_h = omb[(long long)(2 * j) * P + p];
                        off_w = omb[(long long)(2 * j + 1) * P + p];
                        const float mr = omb[(long long)(2 * s.dg * T + j) * P + p];
                        m = 1.f / (1.f + expf(-mr));
                        float2 f = make_float2(0.f, 0.f);   // pre-offset (x, y)
                        if (a.pre) {
                            const float *pp = a.pre + (((long long)b * T + tap) * P + p) * 2;
                            f = make_float2(pp[0], pp[1]);
                        } else if (a.idx) {
                            f = pyramid_flow(a.idx, b, a.gh, a.gw, a.ref_gw, a.pre_scale, p / a.g.Wo, p % a.g.Wo,
                                             tap / s.kw, tap % s.kw);
                        }
                        off_h += f.y;
                        off_w += f.x;
                    } else {
                        off_h = a.offset[((long long)b * 2 * s.dg * T + 2 * j) * P + p];
                        off_w = a.offset[((long long)b * 2 * s.dg * T + 2 * j + 1) * P + p];
                        m = a.mask[((long long)b * s.dg * T + j) * P + p];
                    }
                    float h_im, w_im;
                    if (dcn_sample_point(s, a.g.Wo, tap, p, off_h, off_w, h_im, w_im)) {
                        const DcnCorners c(h_im, w_im, s.H, s.W, s.xs_y, s.xs_x);
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (c.ok[q]) { sp.o[q] = c.o[q]; sp.w[q] = c.w[q]; }
                        sp.m = m;
                    }
                }
                samp[tl * TP + pl] = sp;
            }
            for (int cb0 = 0; cb0 < cpg; cb0 += CB) {
                const int CBn = min(CB, cpg - cb0);
                __syncthreads();
                // ---- bilinear gather into the column tile: row (cl*TB + tl), pixel pl
                const int rows = CBn * TB;
                if (s.xs_c == 1) {
                    // channels-last input: consecutive threads -> consecutive channels of one sample
                    for (int e = t; e < rows * TP; e += 256) {
                        const int cl = e % CBn, rest = e / CBn, pl = rest % TP, tl = rest / TP;
                        const Samp &sp = samp[tl * TP + pl];
                        const float *xc = xb + (g * cpg + cb0 + cl);
                        const float v = dcn_blend(sp.w, xc[sp.o[0]], xc[sp.o[1]], xc[sp.o[2]], xc[sp.o[3]]);
                        col[(cl * TB + tl) * TP + pl] = v * sp.m;
                    }
                } else {
                    for (int e = t; e < rows * TP; e += 256) {
                        const int pl = e % TP, row = e / TP, cl = row / TB, tl = row % TB;
                        const Samp &sp = samp[tl * TP + pl];
                        const float *xc = xb + (long long)(g * cpg + cb0 + cl) * s.xs_c;
                        const float v = dcn_blend(sp.w, xc[sp.o[0]], xc[sp.o[1]], xc[sp.o[2]], xc[sp.o[3]]);
                        col[row * TP + pl] = v * sp.m;
                    }
                }
                // ---- contraction over this K slice, KSUB rows of weights at a time
                for (int k0 = 0; k0 < rows; k0 += KSUB) {
                    const int kn = min(KSUB, rows - k0);
                    __syncthreads();
                    for (int e = t; e < KSUB * NOUT; e += 256) {
                        const int kk = e % KSUB, o = e / KSUB;
                        float wv = 0.f;
                        if (kk < kn && o0 + o < s.Cout) {
                            const int row = k0 + kk, cl = row / TB, tl = row % TB;
                            wv = a.weight[((long long)(o0 + o) * s.C + g * cpg + cb0 + cl) * T + t0 + tl];
                        }
                        Ws[kk * NOUT + o] = wv;
                    }
                    __syncthreads();
#pragma unroll 4
                    for (int kk = 0; kk < kn; ++kk) {
                        const float4 cv = *reinterpret_cast<const float4 *>(&col[(k0 + kk) * TP + tx * 4]);
#pragma unroll
                        for (int i = 0; i < NO; ++i) {
                            const float wv = Ws[kk * NOUT + ty + 16 * i];
                            acc[i][0] = fmaf(wv, cv.x, acc[i][0]);
                            acc[i][1] = fmaf(wv, cv.y, acc[i][1]);
                            acc[i][2] = fmaf(wv, cv.z, acc[i][2]);
                            acc[i][3] = fmaf(wv, cv.w, acc[i][3]);
                        }
                    }
                }
            }
        }
    }
    // ---- epilogue: bias, optional LeakyReLU, store
    float *ob = a.out + (long long)b * s.os_b;
#pragma unroll
    for (int i = 0; i < NO; ++i) {
        const int o = o0 + ty + 16 * i;
        if (o >= s.Cout) continue;
        const float bv = a.bias ? a.bias[o] : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int p = p0 + tx * 4 + j;
            if (p >= P) continue;
            float v = acc[i][j] + bv;
            if (a.slope != 1.f) v = v > 0.f ? v : v * a.slope;
            ob[(long long)o * s.os_c + (long long)(p / a.g.Wo) * s.os_y + (long long)(p % a.g.Wo) * s.os_x] = v;
        }
    }
}

template <int NO>
static int launch_no(const DcnArgs &a, cudaStream_t st) {
    const int NOUT = 16 * NO;
    const size_t smem = sizeof(Samp) * MAXT * TP + (size_t)a.CB * MAXT * TP * 4 + (size_t)KSUB * NOUT * 4;
    C2M_CUDA(cudaFuncSetAttribute(dcn_fwd_kernel<NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ceil_div(a.g.Ho * a.g.Wo, TP), a.s.B, ceil_div(a.s.Cout, NOUT));
    dcn_fwd_kernel<NO><<<grid, 256, smem, st>>>(a);
    C2M_LAUNCH_CHECK("dcn_fwd_kernel");
    return C2M_OK;
}

static int dcn_launch(DcnArgs a, cudaStream_t st) {
    const c2m_dcn_shape &s = a.s;
    C2M_CHECK_ARG(s.Cout > 0, "dcn_v2: empty tensor");
    if (int rc = dcn_geometry(&s, "dcn_v2", a.g)) return rc;
    a.CB = a.g.cpg < MAXCB ? a.g.cpg : MAXCB;
    if (s.Cout <= 16) return launch_no<1>(a, st);
    if (s.Cout <= 32) return launch_no<2>(a, st);
    if (s.Cout <= 64) return launch_no<4>(a, st);
    if (s.Cout <= 128) return launch_no<8>(a, st);
    return launch_no<16>(a, st);
}

}  // namespace c2m

extern "C" int c2m_dcn_v2_forward_f32(const float *x, const float *offset, const float *mask, const float *weight,
                                      const float *bias, float *out, const c2m_dcn_shape *shape, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && mask && weight && out && shape, "dcn_v2_forward: null pointer");
    c2m::DcnArgs a = {};
    a.x = x; a.offset = offset; a.mask = mask; a.weight = weight; a.bias = bias; a.out = out;
    a.s = *shape;
    a.slope = 1.f;
    return c2m::dcn_launch(a, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int c2m_dcn_v2_fused_forward_f32(const float *x, const float *om, const float *pre, const int64_t *idx,
                                            int gh, int gw, int ref_gw, int pre_scale, const float *weight,
                                            const float *bias, float lrelu_slope, float *out,
                                            const c2m_dcn_shape *shape, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && om && weight && out && shape, "dcn_v2_fused_forward: null pointer");
    C2M_CHECK_ARG(!(pre == nullptr && idx != nullptr) || (gh > 0 && gw > 0 && ref_gw > 0 && pre_scale > 0),
                  "dcn_v2_fused_forward: idx given without a valid grid/scale");
    c2m::DcnArgs a = {};
    a.x = x; a.om = om; a.pre = pre; a.idx = reinterpret_cast<const long long *>(idx);
    a.gh = gh; a.gw = gw; a.ref_gw = ref_gw; a.pre_scale = pre_scale;
    a.weight = weight; a.bias = bias; a.out = out;
    a.s = *shape;
    a.slope = lrelu_slope;
    return c2m::dcn_launch(a, reinterpret_cast<cudaStream_t>(stream));
}
