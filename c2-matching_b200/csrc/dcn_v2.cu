// Fused (modulated) deformable convolution forward for sm_90a.
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
// The same kernel serves `deform_conv_cuda` (mmsr/models/archs/dcn/src/deform_conv_cuda.cpp): it is templated on
// the scalar type (float, double), takes grouped convolution (weight [Cout, C/groups, kh, kw]) and a null mask
// (modulation 1, DCNv1).
//
// CTA = 256 threads = 64 output pixels x (16*NO) output channels of one conv group; thread (tx,ty) owns pixels
// 4tx..4tx+3 and channels ty+16i.  K is walked over the conv group's input channels in segments that never cross
// a deformable-group boundary (conv groups and deformable groups partition C independently), one channel block at
// a time: the sampling table (4 corner offsets + 4 weights + mask per (tap, pixel)) is computed once per
// (deformable group, tap pass) and shared by all channels of the segment.  A corner outside the image (and every corner
// of a sample outside the window) is stored as offset -1 and reads as exactly 0: like the reference, the gather never
// loads it, so a non-finite element elsewhere in the plane cannot reach the sample through a zero weight.
#include <type_traits>

#include "dcn_sampling.cuh"

namespace c2m {

namespace {
constexpr int TP = 64;        // pixels per CTA
constexpr int MAXT = 9;       // taps per pass

// K rows per weight sub-slice, channels per pass and the widest NO.  fp64 stops at NO = 8 (64 fp64 accumulators per
// thread; wider layers take more z-blocks) and halves the first two: its largest layout (sample table, column tile,
// weight slice at NO = 8) is 32256 + 73728 + 16384 B = 120 KB, where fp32's tile sizes would need 207 KB (fp32 itself
// takes at most 126 KB, at NO = 16).
template <typename T> struct DcnTile { static constexpr int KSUB = 32, MAXCB = 32, MAXNO = 16; };
template <> struct DcnTile<double> { static constexpr int KSUB = 16, MAXCB = 16, MAXNO = 8; };

// CTAs per SM an instantiation is compiled for (0: ptxas' choice).  fp32 NO = 8 keeps the parent kernel's three
// (80 registers); with the conv-group loop state it fits only with its contraction unrolled 2 deep instead of 4.
template <typename T, int NO>
constexpr int dcn_min_ctas() { return sizeof(T) == 4 && NO == 8 ? 3 : 0; }

template <typename T>
struct DcnArgs {
    const T *x, *offset, *mask, *weight, *bias;   // mask == null: modulation 1 (DCNv1)
    const float *om, *pre;                         // fused entry (fp32 only)
    const long long *idx;
    T *out;
    c2m_dcn_shape s;
    DcnGeom g;
    int gh, gw, ref_gw, pre_scale;
    float slope;
    int groups, Cin_g, Cout_g;   // conv groups and channels per conv group, in and out
    int nob;                     // NOUT-channel blocks per conv group
    int CB;                      // channels per pass (<= cpg, <= Cin_g, <= MAXCB)
};

template <typename T>
struct Samp {
    int o[4];
    T w[4];
    T m;
};

__device__ __forceinline__ float dcn_fma(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ double dcn_fma(double a, double b, double c) { return fma(a, b, c); }

// corner value: offset -1 marks a corner the sample does not read
template <typename T>
__device__ __forceinline__ T corner(const T *xc, int o) { return o >= 0 ? xc[o] : (T)0; }

struct Double4 { double x, y, z, w; };
__device__ __forceinline__ float4 col_load4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ Double4 col_load4(const double *p) {
    const double2 lo = reinterpret_cast<const double2 *>(p)[0], hi = reinterpret_cast<const double2 *>(p)[1];
    return {lo.x, lo.y, hi.x, hi.y};
}
}  // namespace

template <typename scalar_t, int NO>
__global__ void __launch_bounds__(256, (dcn_min_ctas<scalar_t, NO>())) dcn_fwd_kernel(const DcnArgs<scalar_t> a) {
    constexpr int KSUB = DcnTile<scalar_t>::KSUB;
    constexpr int KUNROLL = sizeof(scalar_t) == 4 && NO == 8 ? 2 : 4;   // see dcn_min_ctas; the FMA order is the same
    extern __shared__ __align__(16) uint8_t dsm[];
    const c2m_dcn_shape &s = a.s;
    const int T = a.g.T, cpg = a.g.cpg, CB = a.CB;
    const int P = a.g.Ho * a.g.Wo;
    const int NOUT = 16 * NO;

    Samp<scalar_t> *samp = reinterpret_cast<Samp<scalar_t> *>(dsm);                                // [MAXT][TP]
    scalar_t *col = reinterpret_cast<scalar_t *>(dsm + sizeof(Samp<scalar_t>) * MAXT * TP);     // [CB*MAXT][TP]
    scalar_t *Ws = col + (size_t)CB * MAXT * TP;                                                 // [KSUB][NOUT]

    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int b = blockIdx.y, p0 = blockIdx.x * TP;
    const int cg = blockIdx.z / a.nob, ob0 = (blockIdx.z % a.nob) * NOUT;   // conv group, first channel within it
    const int o0 = cg * a.Cout_g + ob0, nout = min(NOUT, a.Cout_g - ob0);   // first output channel, channels here
    const int c_begin = cg * a.Cin_g, c_end = c_begin + a.Cin_g;             // the conv group's input channels
    // weight [o0 + o][c - c_begin][tap] is wbase[(o * Cin_g + c) * T + tap]
    const scalar_t *wbase = a.weight + ((long long)o0 * a.Cin_g - c_begin) * T;
    const scalar_t *xb = a.x + (long long)b * s.xs_b;

    scalar_t acc[NO][4];
#pragma unroll
    for (int i = 0; i < NO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = (scalar_t)0;

    // segments [seg0, seg1) of the conv group's channels, one per deformable group g they meet
    for (int g = c_begin / cpg; g * cpg < c_end; ++g) {
        const int seg0 = max(g * cpg, c_begin), seg1 = min((g + 1) * cpg, c_end);
        for (int t0 = 0; t0 < T; t0 += MAXT) {
            const int TB = min(MAXT, T - t0);
            __syncthreads();
            // ---- sampling table for (tap, pixel), shared by the segment's channels
            for (int e = t; e < TB * TP; e += 256) {
                const int tl = e / TP, pl = e % TP, tap = t0 + tl, p = p0 + pl;
                Samp<scalar_t> sp = {{-1, -1, -1, -1}, {}, (scalar_t)0};
                if (p < P) {
                    const int j = g * T + tap;
                    scalar_t off_h, off_w, m;
                    if (a.om) {
                        if constexpr (std::is_same<scalar_t, float>::value) {
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
                        }
                    } else {
                        off_h = a.offset[((long long)b * 2 * s.dg * T + 2 * j) * P + p];
                        off_w = a.offset[((long long)b * 2 * s.dg * T + 2 * j + 1) * P + p];
                        m = a.mask ? a.mask[((long long)b * s.dg * T + j) * P + p] : (scalar_t)1;
                    }
                    scalar_t h_im, w_im;
                    if (dcn_sample_point(s, a.g.Wo, tap, p, off_h, off_w, h_im, w_im)) {
                        const DcnCorners<scalar_t> c(h_im, w_im, s.H, s.W, s.xs_y, s.xs_x);
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (c.ok[q]) { sp.o[q] = c.o[q]; sp.w[q] = c.w[q]; }
                        sp.m = m;
                    }
                }
                samp[tl * TP + pl] = sp;
            }
            for (int c0 = seg0; c0 < seg1; c0 += CB) {
                const int CBn = min(CB, seg1 - c0);
                __syncthreads();
                // ---- bilinear gather into the column tile: row (cl*TB + tl), pixel pl
                const int rows = CBn * TB;
                if (s.xs_c == 1) {
                    // channels-last input: consecutive threads -> consecutive channels of one sample
                    for (int e = t; e < rows * TP; e += 256) {
                        const int cl = e % CBn, rest = e / CBn, pl = rest % TP, tl = rest / TP;
                        const Samp<scalar_t> &sp = samp[tl * TP + pl];
                        const scalar_t *xc = xb + (c0 + cl);
                        const scalar_t v = dcn_blend(sp.w, corner(xc, sp.o[0]), corner(xc, sp.o[1]), corner(xc, sp.o[2]),
                                                     corner(xc, sp.o[3]));
                        col[(cl * TB + tl) * TP + pl] = v * sp.m;
                    }
                } else {
                    for (int e = t; e < rows * TP; e += 256) {
                        const int pl = e % TP, row = e / TP, cl = row / TB, tl = row % TB;
                        const Samp<scalar_t> &sp = samp[tl * TP + pl];
                        const scalar_t *xc = xb + (long long)(c0 + cl) * s.xs_c;
                        const scalar_t v = dcn_blend(sp.w, corner(xc, sp.o[0]), corner(xc, sp.o[1]), corner(xc, sp.o[2]),
                                                     corner(xc, sp.o[3]));
                        col[row * TP + pl] = v * sp.m;
                    }
                }
                // ---- contraction over this K slice, KSUB rows of weights at a time
                for (int k0 = 0; k0 < rows; k0 += KSUB) {
                    const int kn = min(KSUB, rows - k0);
                    __syncthreads();
                    for (int e = t; e < KSUB * NOUT; e += 256) {
                        const int kk = e % KSUB, o = e / KSUB;
                        scalar_t wv = (scalar_t)0;
                        if (kk < kn && o < nout) {
                            const int row = k0 + kk, cl = row / TB, tl = row % TB;
                            wv = wbase[((long long)o * a.Cin_g + c0 + cl) * T + t0 + tl];
                        }
                        Ws[kk * NOUT + o] = wv;
                    }
                    __syncthreads();
#pragma unroll(KUNROLL)
                    for (int kk = 0; kk < kn; ++kk) {
                        const auto cv = col_load4(&col[(k0 + kk) * TP + tx * 4]);
#pragma unroll
                        for (int i = 0; i < NO; ++i) {
                            const scalar_t wv = Ws[kk * NOUT + ty + 16 * i];
                            acc[i][0] = dcn_fma(wv, cv.x, acc[i][0]);
                            acc[i][1] = dcn_fma(wv, cv.y, acc[i][1]);
                            acc[i][2] = dcn_fma(wv, cv.z, acc[i][2]);
                            acc[i][3] = dcn_fma(wv, cv.w, acc[i][3]);
                        }
                    }
                }
            }
        }
    }
    // ---- epilogue: bias, optional LeakyReLU, store
    scalar_t *ob = a.out + (long long)b * s.os_b;
#pragma unroll
    for (int i = 0; i < NO; ++i) {
        if (ty + 16 * i >= nout) continue;
        const int o = o0 + ty + 16 * i;
        const scalar_t bv = a.bias ? a.bias[o] : (scalar_t)0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int p = p0 + tx * 4 + j;
            if (p >= P) continue;
            scalar_t v = acc[i][j] + bv;
            if (a.slope != 1.f) v = v > (scalar_t)0 ? v : v * (scalar_t)a.slope;
            ob[(long long)o * s.os_c + (long long)(p / a.g.Wo) * s.os_y + (long long)(p % a.g.Wo) * s.os_x] = v;
        }
    }
}

template <typename scalar_t, int NO>
static int launch_no(DcnArgs<scalar_t> a, cudaStream_t st) {
    const int NOUT = 16 * NO;
    const size_t smem = sizeof(Samp<scalar_t>) * MAXT * TP + (size_t)a.CB * MAXT * TP * sizeof(scalar_t) +
                        (size_t)DcnTile<scalar_t>::KSUB * NOUT * sizeof(scalar_t);
    a.nob = ceil_div(a.Cout_g, NOUT);
    C2M_CHECK_ARG((long long)a.groups * a.nob <= 65535 && a.s.B <= 65535, "deformable convolution: grid too large "
                  "(%d images, %d groups x %d channel blocks)", a.s.B, a.groups, a.nob);
    C2M_CUDA(cudaFuncSetAttribute(dcn_fwd_kernel<scalar_t, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ceil_div(a.g.Ho * a.g.Wo, TP), a.s.B, a.groups * a.nob);
    dcn_fwd_kernel<scalar_t, NO><<<grid, 256, smem, st>>>(a);
    C2M_LAUNCH_CHECK("dcn_fwd_kernel");
    return C2M_OK;
}

// NO from the output channels of one conv group
template <typename scalar_t>
static int dcn_launch(DcnArgs<scalar_t> a, const char *who, cudaStream_t st) {
    const c2m_dcn_shape &s = a.s;
    C2M_CHECK_ARG(s.Cout > 0, "%s: empty tensor", who);
    if (int rc = dcn_geometry(&s, who, a.g)) return rc;
    C2M_CHECK_ARG(a.groups > 0 && s.C % a.groups == 0 && s.Cout % a.groups == 0,
                  "%s: input channels (%d) and output channels (%d) must be divisible by groups (%d)", who, s.C,
                  s.Cout, a.groups);
    a.Cin_g = s.C / a.groups;
    a.Cout_g = s.Cout / a.groups;
    a.CB = min(min(a.g.cpg, a.Cin_g), DcnTile<scalar_t>::MAXCB);
    if (a.Cout_g <= 16) return launch_no<scalar_t, 1>(a, st);
    if (a.Cout_g <= 32) return launch_no<scalar_t, 2>(a, st);
    if (a.Cout_g <= 64) return launch_no<scalar_t, 4>(a, st);
    if constexpr (DcnTile<scalar_t>::MAXNO == 8) {
        return launch_no<scalar_t, 8>(a, st);
    } else {
        if (a.Cout_g <= 128) return launch_no<scalar_t, 8>(a, st);
        return launch_no<scalar_t, 16>(a, st);
    }
}

template <typename scalar_t>
static int deform_forward(const scalar_t *x, const scalar_t *offset, const scalar_t *mask, const scalar_t *weight,
                          const scalar_t *bias, int groups, scalar_t *out, const c2m_dcn_shape *shape,
                          c2m_stream_t stream) {
    DcnArgs<scalar_t> a = {};
    a.x = x; a.offset = offset; a.mask = mask; a.weight = weight; a.bias = bias; a.out = out;
    a.s = *shape;
    a.slope = 1.f;
    a.groups = groups;
    return dcn_launch(a, "deform_conv", reinterpret_cast<cudaStream_t>(stream));
}

}  // namespace c2m

extern "C" int c2m_deform_conv_forward_f32(const float *x, const float *offset, const float *mask,
                                           const float *weight, const float *bias, int groups, float *out,
                                           const c2m_dcn_shape *shape, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && weight && out && shape, "deform_conv_forward: null pointer");
    return c2m::deform_forward(x, offset, mask, weight, bias, groups, out, shape, stream);
}

extern "C" int c2m_deform_conv_forward_f64(const double *x, const double *offset, const double *mask,
                                           const double *weight, const double *bias, int groups, double *out,
                                           const c2m_dcn_shape *shape, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && offset && weight && out && shape, "deform_conv_forward: null pointer");
    return c2m::deform_forward(x, offset, mask, weight, bias, groups, out, shape, stream);
}

extern "C" int c2m_dcn_v2_fused_forward_f32(const float *x, const float *om, const float *pre, const int64_t *idx,
                                            int gh, int gw, int ref_gw, int pre_scale, const float *weight,
                                            const float *bias, float lrelu_slope, float *out,
                                            const c2m_dcn_shape *shape, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && om && weight && out && shape, "dcn_v2_fused_forward: null pointer");
    C2M_CHECK_ARG(!(pre == nullptr && idx != nullptr) || (gh > 0 && gw > 0 && ref_gw > 0 && pre_scale > 0),
                  "dcn_v2_fused_forward: idx given without a valid grid/scale");
    c2m::DcnArgs<float> a = {};
    a.x = x; a.om = om; a.pre = pre; a.idx = reinterpret_cast<const long long *>(idx);
    a.gh = gh; a.gw = gw; a.ref_gw = ref_gw; a.pre_scale = pre_scale;
    a.weight = weight; a.bias = bias; a.out = out;
    a.s = *shape;
    a.slope = lrelu_slope;
    a.groups = 1;
    return c2m::dcn_launch(a, "dcn_v2", reinterpret_cast<cudaStream_t>(stream));
}
