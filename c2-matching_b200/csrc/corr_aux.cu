// Correlation support kernels: layout/normalise/split prep, Ref patch norms, the generic
// CUDA-core candidate search (any patch size / stride / channel count) and the exact rescoring
// pass that produces the final index map.  See corr_internal.cuh for the HBM layouts.
//
// Reference semantics restated: mmsr/models/archs/ref_map_util.py:26-86 (feature_match_index) and
// mmsr/models/archs/corres_generation_arch.py:56-58 (F.normalize over channels).
#include <cfloat>
#include <cstdlib>
#include "corr_internal.cuh"

namespace c2m {

// ------------------------------------------------------------------------------------------
// largest finite |x| of each image -> scale exponent so that |x| * 2^sexp <= 1024 (fp16-safe with 5 bits of
// headroom below 65504).  Elements far below amax still reach the fp16 subnormals, whose absolute rounding the
// rescoring window covers separately (c_abi.cu, DESIGN.md K2).  NaN / Inf are left out of the maximum (their
// pixels are flagged and scored exactly), so one Inf does not push the finite elements out of fp16's range.
// ------------------------------------------------------------------------------------------
// max finite |x| of image blockIdx.y as float bits (atomicMax on the bits of non-negative floats orders like the
// values); out_bits[b] starts at 0
__global__ void amax_kernel(const float *__restrict__ x, size_t n, unsigned *__restrict__ out_bits) {
    const float *xb = x + blockIdx.y * n;
    float m = 0.f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float a = fabsf(xb[i]);
        if (a < INFINITY) m = fmaxf(m, a);        // false for NaN and Inf
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out_bits + blockIdx.y, __float_as_uint(m));
}

// sexp[b] in [-126, 126], so that 2^sexp and 2^-sexp are normal floats (a map whose largest finite |x| is below
// 2^-116 keeps less than 10 bits of fp16 headroom; the window's subnormal term covers its rounding).  After l2norm
// |x| / max(||x||, 1e-12) <= min(1, amax 1e12): 1 (sexp = 10) unless every pixel norm is below 1e-12, where the
// normalised map is the input times 1e12 and takes that map's exponent.
__global__ void sexp_kernel(const unsigned *__restrict__ amax_bits, int *__restrict__ sexp, int B, int l2norm) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float a = __uint_as_float(amax_bits[b]);
    if (l2norm) a = fminf(1.f, a * 1e12f);
    int e = 0;
    if (a > 0.f) frexpf(a, &e);                  // a = f * 2^e, f in [0.5,1)  =>  a <= 2^e
    sexp[b] = min(126, max(-126, 10 - e));
}

// ------------------------------------------------------------------------------------------
// prep: NCHW fp32 -> p32 / hi / lo / ss.   One block = 32 consecutive pixels of one image.
// 256 threads; channel blocks of 64 go through a padded smem tile so that both the NCHW reads
// (32 consecutive pixels of one channel) and the pixel-major writes are coalesced.
// ------------------------------------------------------------------------------------------
constexpr int PREP_PIX = 32;
constexpr int PREP_CB = 64;

__global__ void __launch_bounds__(256) prep_kernel(const float *__restrict__ x, int C, int Cp, int HW, int l2norm,
                                                   const int *__restrict__ sexp_p, float *__restrict__ p32,
                                                   __half *__restrict__ hi, __half *__restrict__ lo,
                                                   float *__restrict__ ss) {
    __shared__ float tile[PREP_CB][PREP_PIX + 1];
    __shared__ float red[8][PREP_PIX];
    __shared__ float ss_s[PREP_PIX];

    const int b = blockIdx.y;
    const int pix0 = blockIdx.x * PREP_PIX;
    const int t = threadIdx.x;
    const int lp = t & 31, lg = t >> 5;          // load mapping: pixel fastest
    const float *xb = x + (size_t)b * C * HW;
    const bool pv = pix0 + lp < HW;

    // pass 1: per-pixel L2 norm over channels (F.normalize(dim=0): x / max(||x||_2, 1e-12))
    float nrm = 1.f;
    if (l2norm) {
        float acc = 0.f;
        for (int c = lg; c < C; c += 8) {
            float v = pv ? xb[(size_t)c * HW + pix0 + lp] : 0.f;
            acc = fmaf(v, v, acc);
        }
        red[lg][lp] = acc;
        __syncthreads();
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += red[i][lp];
        nrm = fmaxf(sqrtf(s), 1e-12f);
    }
    if (t < PREP_PIX) ss_s[t] = 0.f;
    const float S = ldexpf(1.f, sexp_p[b]);

    const int wp = t & 31, wq = t >> 5;          // hi/lo write mapping: pixel fastest, octet = wq
    const int rp = t >> 3, rq = t & 7;           // p32 write mapping: 8 threads per pixel
    float ssacc = 0.f;
    for (int c0 = 0; c0 < Cp; c0 += PREP_CB) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < PREP_CB / 8; ++i) {
            const int c = c0 + lg + i * 8;
            float v = 0.f;
            if (pv && c < C) {
                v = xb[(size_t)c * HW + pix0 + lp];
                if (l2norm) v = v / nrm;
            }
            tile[lg + i * 8][lp] = v;
        }
        __syncthreads();
        // p32 [pix][Cp]
        if (pix0 + rp < HW && c0 + rq * 8 < Cp) {
            float4 a, bq;
            a.x = tile[rq * 8 + 0][rp]; a.y = tile[rq * 8 + 1][rp]; a.z = tile[rq * 8 + 2][rp]; a.w = tile[rq * 8 + 3][rp];
            bq.x = tile[rq * 8 + 4][rp]; bq.y = tile[rq * 8 + 5][rp]; bq.z = tile[rq * 8 + 6][rp]; bq.w = tile[rq * 8 + 7][rp];
            float4 *dst = reinterpret_cast<float4 *>(p32 + ((size_t)b * HW + pix0 + rp) * Cp + c0 + rq * 8);
            dst[0] = a;
            dst[1] = bq;
        }
        // hi / lo [Cp/8][HW][8]
        if (pix0 + wp < HW && c0 + wq * 8 < Cp) {
            __align__(16) __half h8[8];
            __align__(16) __half l8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v = tile[wq * 8 + j][wp] * S;
                ssacc = fmaf(v, v, ssacc);                  // non-finite iff the pixel holds NaN / Inf
                psa_split(isfinite(v) ? v : 0.f, h8[j], l8[j]);
            }
            const size_t o = (((size_t)b * (Cp / 8) + (c0 / 8 + wq)) * HW + pix0 + wp) * 8;
            *reinterpret_cast<uint4 *>(hi + o) = *reinterpret_cast<const uint4 *>(h8);
            *reinterpret_cast<uint4 *>(lo + o) = *reinterpret_cast<const uint4 *>(l8);
        }
    }
    atomicAdd(&ss_s[wp], ssacc);
    __syncthreads();
    if (t < PREP_PIX && pix0 + t < HW) ss[(size_t)b * HW + pix0 + t] = ss_s[t];
}

int corr_prep_launch(const float *x, int B, int C, int Cp, int HW, int l2norm, int map_slot,
                     const CorrWorkspace &ws, float *p32, __half *hi, __half *lo, float *ss, cudaStream_t st) {
    const size_t n = (size_t)C * HW;
    int blocks = (int)((n + 1023) / 1024);
    const int cap = ceil_div(1184, B);
    if (blocks > cap) blocks = cap;
    amax_kernel<<<dim3(blocks, B), 256, 0, st>>>(x, n, ws.amax_bits + map_slot * B);
    C2M_LAUNCH_CHECK("amax_kernel");
    sexp_kernel<<<ceil_div(B, 256), 256, 0, st>>>(ws.amax_bits + map_slot * B, ws.sexp + map_slot * B, B, l2norm);
    C2M_LAUNCH_CHECK("sexp_kernel");
    dim3 grid(ceil_div(HW, PREP_PIX), B);
    prep_kernel<<<grid, 256, 0, st>>>(x, C, Cp, HW, l2norm, ws.sexp + map_slot * B, p32, hi, lo, ss);
    C2M_LAUNCH_CHECK("prep_kernel");
    return C2M_OK;
}

// ------------------------------------------------------------------------------------------
// Ref column scale in search units (corr_internal.cuh), from the scaled ss:
//     rinv[b][r] = 1 / (||P_r|| 2^sr + 1e-5 2^sr) = 2^-sr / (||P_r|| + 1e-5)      (ref_map_util.py:63), 1 for raw scores
// Neither factor leaves fp32's range (||P_r|| 2^sr <= 3 sqrt(C) 1024, sr in [-126, 126]).  A patch holding a
// non-finite element gets NaN and goes to the list that the rescoring scores exactly for every query.
// ------------------------------------------------------------------------------------------
__global__ void rinv_kernel(const float *__restrict__ ss, float *__restrict__ rinv, int hr, int wr, int rh, int rw,
                            int patch, int s_ref, int is_norm, const int *__restrict__ sexp_ref,
                            unsigned *__restrict__ pr_max_bits, unsigned *__restrict__ rinv_max_bits,
                            int *__restrict__ flag_ref, unsigned *__restrict__ flag_count) {
    const int b = blockIdx.y;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float pn = 0.f, rv = 0.f;
    if (r < rh * rw) {
        const int ry = (r / rw) * s_ref, rx = (r % rw) * s_ref;
        const float *s = ss + (size_t)b * hr * wr;
        float acc = 0.f;
        for (int dy = 0; dy < patch; ++dy)
            for (int dx = 0; dx < patch; ++dx) acc += s[(ry + dy) * wr + rx + dx];
        float ri;
        if (isfinite(acc)) {
            const float nrm = sqrtf(acc);
            ri = is_norm ? fminf(1.f / (nrm + ldexpf(1e-5f, sexp_ref[b])), FLT_MAX) : 1.f;
            pn = nrm * ri;               // <= 1 when is_norm: ~1e-14 for a Ref map at 1e-20 (the +1e-5 dominates)
            if (nrm > 0.f) rv = ri;      // an all-zero patch rounds exactly: it must not widen the window
        } else {
            ri = __int_as_float(0x7fffffff);
            flag_ref[(size_t)b * rh * rw + atomicAdd(flag_count + b, 1u)] = r;
        }
        rinv[(size_t)b * rh * rw + r] = ri;
    }
    // largest ||P_r|| rinv_r of the image (the scaled patch norm for raw scores): the Ref factor of the image's score
    // scale, which every term of the rescoring window carries; largest rinv of a nonzero Ref patch: scales the absolute
    // (fp16 subnormal) rounding of the Ref operand
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        pn = fmaxf(pn, __shfl_xor_sync(0xffffffffu, pn, o));
        rv = fmaxf(rv, __shfl_xor_sync(0xffffffffu, rv, o));
    }
    if ((threadIdx.x & 31) == 0 && pn > 0.f) atomicMax(pr_max_bits + b, __float_as_uint(pn));
    if ((threadIdx.x & 31) == 0 && rv > 0.f) atomicMax(rinv_max_bits + b, __float_as_uint(rv));
}

int corr_rinv_launch(const CorrGeom &g, const CorrWorkspace &ws, int is_norm, cudaStream_t st) {
    dim3 grid(ceil_div(g.NR, 256), g.B);
    rinv_kernel<<<grid, 256, 0, st>>>(ws.ss_ref, ws.rinv, g.hr, g.wr, g.rh, g.rw, g.patch, g.s_ref, is_norm, ws.sexp + g.B,
                                       ws.pr_max_bits, ws.rinv_max_bits, ws.flag_ref, ws.flag_count);
    C2M_LAUNCH_CHECK("rinv_kernel");
    return C2M_OK;
}

// ------------------------------------------------------------------------------------------
// Generic candidate search on CUDA cores (fp32 FFMA): any patch size, strides, channel count.
// Block = 64 queries x (all Ref patches of one chunk), 64x64 score tiles, 4x4 per thread,
// K streamed 8 channels of one tap at a time.  Emits the same Candidate partials as the
// tensor-core search; the final answer always comes from the rescoring pass.  It multiplies the
// operands scaled by their image's 2^sexp (<= 1024, so no product overflows; a non-finite element
// reads as 0, its patches are scored exactly), for scores in search units like the tensor cores'.
// ------------------------------------------------------------------------------------------
constexpr int GS_T = 64;

__device__ __forceinline__ float scaled_operand(float v, float S) {
    v *= S;
    return isfinite(v) ? v : 0.f;
}

__global__ void __launch_bounds__(256) search_generic_kernel(const float *__restrict__ pin, const float *__restrict__ pref,
                                                             const float *__restrict__ rinv, const int *__restrict__ sexp,
                                                             Candidate *__restrict__ part, CorrGeom g, int nchunk) {
    __shared__ __align__(16) float As[8][GS_T + 4];
    __shared__ __align__(16) float Bs[8][GS_T + 4];
    __shared__ int qpix[GS_T];
    __shared__ int rpix[GS_T];
    __shared__ float rsc[GS_T];
    struct Red { float v[GEN_TOPK]; int i[GEN_TOPK]; float dropped; };      // 36 B
    __shared__ Red red[GS_T][16];

    const int b = blockIdx.z, chunk = blockIdx.y;
    const int q0 = blockIdx.x * GS_T;
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const float *pinb = pin + (size_t)b * g.h * g.w * g.Cp;
    const float *prefb = pref + (size_t)b * g.hr * g.wr * g.Cp;
    const float *rinvb = rinv + (size_t)b * g.NR;
    const float S = ldexpf(1.f, sexp[t < 128 ? b : g.B + b]);      // loader: threads 0..127 query, 128..255 Ref

    if (t < GS_T) {
        const int q = q0 + t;
        qpix[t] = q < g.NQ ? ((q / g.gw) * g.s_in) * g.w + (q % g.gw) * g.s_in : -1;
    }
    const int per = ceil_div(ceil_div(g.NR, GS_T), nchunk) * GS_T;
    const int r_begin = chunk * per, r_end = min(g.NR, r_begin + per);

    float cv[4][GEN_TOPK], cdrop[4];
    int ci[4][GEN_TOPK];
#pragma unroll
    for (int i = 0; i < 4; ++i) { cand_init(cv[i], ci[i]); cdrop[i] = -INFINITY; }

    const int lrow = t >> 1 & 63, lhalf = t & 1;     // loader: threads 0..127 -> A, 128..255 -> B
    for (int r0 = r_begin; r0 < r_end; r0 += GS_T) {
        __syncthreads();
        if (t < GS_T) {
            const int r = r0 + t;
            const bool ok = r < r_end;
            rpix[t] = ok ? ((r / g.rw) * g.s_ref) * g.wr + (r % g.rw) * g.s_ref : -1;
            rsc[t] = ok ? rinvb[r] : 0.f;
        }
        __syncthreads();
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

        for (int tap = 0; tap < g.patch * g.patch; ++tap) {
            const int dy = tap / g.patch, dx = tap % g.patch;
            for (int c0 = 0; c0 < g.Cp; c0 += 8) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t < 128) {
                    const int pq = qpix[lrow];
                    if (pq >= 0) v = *reinterpret_cast<const float4 *>(pinb + (size_t)(pq + dy * g.w + dx) * g.Cp + c0 + lhalf * 4);
                } else {
                    const int pr = rpix[lrow];
                    if (pr >= 0) v = *reinterpret_cast<const float4 *>(prefb + (size_t)(pr + dy * g.wr + dx) * g.Cp + c0 + lhalf * 4);
                }
                __syncthreads();
                float(*dst)[GS_T + 4] = t < 128 ? As : Bs;
                dst[lhalf * 4 + 0][lrow] = scaled_operand(v.x, S);
                dst[lhalf * 4 + 1][lrow] = scaled_operand(v.y, S);
                dst[lhalf * 4 + 2][lrow] = scaled_operand(v.z, S);
                dst[lhalf * 4 + 3][lrow] = scaled_operand(v.w, S);
                __syncthreads();
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
                    const float4 bb = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
                    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = r0 + tx * 4 + j;
            if (r < r_end) {
                const float sc = rsc[tx * 4 + j];
#pragma unroll
                for (int i = 0; i < 4; ++i) cand_push(acc[i][j] * sc, r, cv[i], ci[i], cdrop[i]);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        Red c;
#pragma unroll
        for (int k = 0; k < GEN_TOPK; ++k) { c.v[k] = cv[i][k]; c.i[k] = ci[i][k]; }
        c.dropped = cdrop[i];
        red[ty * 4 + i][tx] = c;
    }
    __syncthreads();
    if (t < GS_T && q0 + t < g.NQ) {
        float av[GEN_TOPK], adrop = -INFINITY;
        int ai[GEN_TOPK];
        cand_init(av, ai);
        for (int k = 0; k < 16; ++k) {
            const Red c = red[t][k];
            adrop = fmaxf(adrop, c.dropped);
#pragma unroll
            for (int j = 0; j < GEN_TOPK; ++j)
                if (c.i[j] != 0x7fffffff) cand_push(c.v[j], c.i[j], av, ai, adrop);
        }
        part[((size_t)b * nchunk + chunk) * g.NQ + q0 + t] = cand_pack(av, ai, adrop);
    }
}

void corr_generic_chunk_geom(const CorrGeom &g, int nchunk, CorrChunkGeom &cg) {
    cg.mode = 0;
    cg.per = ceil_div(ceil_div(g.NR, GS_T), nchunk) * GS_T;       // same split as search_generic_kernel
    cg.n_rt = cg.rt_x = cg.tile_rows = cg.tile_cols = 0;
}

int corr_search_generic_launch(const CorrGeom &g, const CorrWorkspace &ws, cudaStream_t st) {
    dim3 grid(ceil_div(g.NQ, GS_T), ws.nchunk, g.B);
    search_generic_kernel<<<grid, 256, 0, st>>>(ws.p32_in, ws.p32_ref, ws.rinv, ws.sexp, ws.part, g, ws.nchunk);
    C2M_LAUNCH_CHECK("search_generic_kernel");
    return C2M_OK;
}

// ------------------------------------------------------------------------------------------
// Exact rescoring.  The searches rank Ref patches by an APPROXIMATE score s~ (tensor-core / fp32-FMA rounding);
// the index map is defined on the exact one,
//     s(r) = float( sum_k double(q[k]) * double( float(ref[k] / (float(sqrt(ss_r)) + 1e-5f)) ) )
// — the reference's arithmetic (Ref patch normalised in fp32 first, ref_map_util.py:63) with an error-free
// accumulation.  With |s~(r) - s(r)| <= E for every r (E = window/2, DESIGN.md K2 derives it from the number of
// accumulation steps, the operand split and the absolute rounding of fp16-subnormal operand elements), the exact argmax r* satisfies s~(r*) >= max s~ - 2E, so it is enough
// to rescore every candidate inside that window.  The searches keep a top-2 per (query, Ref chunk): the list of a
// chunk is COMPLETE unless its second entry is itself inside the window (then a third one could be hiding); those
// (query, chunk) pairs go to an overflow list and `rescore_overflow_kernel` re-scans the whole chunk exactly.
// Hence idx/val equal the exhaustive exact result, whatever the tensor cores rounded.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// exact score of (query pixel qp, Ref pixel rp), computed by one warp; every lane returns it.  Rows are read
// as float4 (Cp is a multiple of 8) with the tap / channel loops unrolled so that several loads are in flight.
__device__ __noinline__ float exact_score_warp(const float *__restrict__ pinb, const float *__restrict__ prefb,
                                               const CorrGeom &g, int qp, int rp, int is_norm, int lane) {
    const int taps = g.patch * g.patch;
    float denom = 1.f;
    if (is_norm) {
        double ss = 0.0;
#pragma unroll 3
        for (int tap = 0; tap < taps; ++tap) {
            const float *row = prefb + (size_t)(rp + (tap / g.patch) * g.wr + tap % g.patch) * g.Cp;
#pragma unroll 2
            for (int c = lane * 4; c < g.Cp; c += 128) {
                const float4 v = *reinterpret_cast<const float4 *>(row + c);
                ss += (double)v.x * (double)v.x;
                ss += (double)v.y * (double)v.y;
                ss += (double)v.z * (double)v.z;
                ss += (double)v.w * (double)v.w;
            }
        }
        ss = warp_sum(ss);
        denom = (float)sqrt(ss) + 1e-5f;
    }
    double acc = 0.0;
#pragma unroll 3
    for (int tap = 0; tap < taps; ++tap) {
        const int dy = tap / g.patch, dx = tap % g.patch;
        const float *rrow = prefb + (size_t)(rp + dy * g.wr + dx) * g.Cp;
        const float *qrow = pinb + (size_t)(qp + dy * g.w + dx) * g.Cp;
#pragma unroll 2
        for (int c = lane * 4; c < g.Cp; c += 128) {
            const float4 rv = *reinterpret_cast<const float4 *>(rrow + c);
            const float4 qv = *reinterpret_cast<const float4 *>(qrow + c);
            acc += (double)qv.x * (double)(is_norm ? __fdiv_rn(rv.x, denom) : rv.x);
            acc += (double)qv.y * (double)(is_norm ? __fdiv_rn(rv.y, denom) : rv.y);
            acc += (double)qv.z * (double)(is_norm ? __fdiv_rn(rv.z, denom) : rv.z);
            acc += (double)qv.w * (double)(is_norm ? __fdiv_rn(rv.w, denom) : rv.w);
        }
    }
    return (float)warp_sum(acc);
}

// fp32 FMA score in search units of (query pixel qp, Ref pixel rp): the operands scaled by Sq = 2^sexp_in, Sr =
// 2^sexp_ref of their image (finite ones <= 1024: no product overflows), times the Ref column scale rinv_r; one warp.
// Differs from the exact score (in search units) by at most E32 = (K + 8) 2^-24 ||P_q|| ||P_r|| rinv_r (K-term FMA
// chain + the reciprocal instead of the per-element division), plus the tiny absolute term of products and elements
// that underflow (`tiny_coef`).  ~1/8 of the instructions of exact_score_warp: a prefilter, never a result.
__device__ __noinline__ float fp32_score_warp(const float *__restrict__ pinb, const float *__restrict__ prefb,
                                              const CorrGeom &g, int qp, int rp, float rinv_r, float Sq, float Sr,
                                              int lane) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 3
    for (int tap = 0; tap < g.patch * g.patch; ++tap) {
        const int dy = tap / g.patch, dx = tap % g.patch;
        const float *rrow = prefb + (size_t)(rp + dy * g.wr + dx) * g.Cp;
        const float *qrow = pinb + (size_t)(qp + dy * g.w + dx) * g.Cp;
#pragma unroll 2
        for (int c = lane * 4; c < g.Cp; c += 128) {
            const float4 rv = *reinterpret_cast<const float4 *>(rrow + c);
            const float4 qv = *reinterpret_cast<const float4 *>(qrow + c);
            a0 = fmaf(qv.x * Sq, rv.x * Sr, a0); a1 = fmaf(qv.y * Sq, rv.y * Sr, a1);
            a2 = fmaf(qv.z * Sq, rv.z * Sr, a2); a3 = fmaf(qv.w * Sq, rv.w * Sr, a3);
        }
    }
    float s32 = (a0 + a1) + (a2 + a3);
#pragma unroll
    for (int of = 16; of; of >>= 1) s32 += __shfl_xor_sync(0xffffffffu, s32, of);
    return s32 * rinv_r;
}

__device__ __forceinline__ double query_patch_ss(const float *__restrict__ pinb, const CorrGeom &g, int qp, int lane) {
    double ssq = 0.0;
#pragma unroll 3
    for (int tap = 0; tap < g.patch * g.patch; ++tap) {
        const float *row = pinb + (size_t)(qp + (tap / g.patch) * g.w + tap % g.patch) * g.Cp;
#pragma unroll 2
        for (int c = lane * 4; c < g.Cp; c += 128) {
            const float4 v = *reinterpret_cast<const float4 *>(row + c);
            ssq += (double)v.x * (double)v.x + (double)v.y * (double)v.y;
            ssq += (double)v.z * (double)v.z + (double)v.w * (double)v.w;
        }
    }
    return warp_sum(ssq);
}

// The per-image quantities of the window, in search units (corr_internal.cuh): u, the operand scales, and the
// Ref-side factors P (the largest ||P_r|| rinv_r of the image: the scaled patch norm for raw scores, at most 1 and
// far below it for a Ref map small against the reference's + 1e-5 when normalised) and R (the largest rinv of a
// nonzero Ref patch, or 1 for raw scores).  ||P_q|| P bounds every |score| of the query.
struct ImageScale {
    int u;
    float Sq, Sr, P, R;
};
__device__ __forceinline__ ImageScale image_scale(const int *__restrict__ sexp, const unsigned *__restrict__ pr_max_bits,
                                                  const unsigned *__restrict__ rinv_max_bits, int B, int b, int is_norm) {
    ImageScale s;
    const int sq = sexp[b], sr = sexp[B + b];
    s.u = is_norm ? sq : sq + sr;
    s.Sq = ldexpf(1.f, sq);
    s.Sr = ldexpf(1.f, sr);
    s.P = __uint_as_float(pr_max_bits[b]);
    s.R = is_norm ? __uint_as_float(rinv_max_bits[b]) : 1.f;
    return s;
}

__global__ void __launch_bounds__(256) rescore_kernel(const float *__restrict__ pin, const float *__restrict__ pref,
                                                      const Candidate *__restrict__ part, CorrGeom g, int nchunk,
                                                      float window_coef, float sub_coef, float e32_coef, float tiny_coef,
                                                      const float *__restrict__ rinv,
                                                      const unsigned *__restrict__ pr_max_bits,
                                                      const unsigned *__restrict__ rinv_max_bits,
                                                      const int *__restrict__ sexp, int is_norm,
                                                      const int *__restrict__ flag_ref,
                                                      const unsigned *__restrict__ flag_count,
                                                      unsigned long long *__restrict__ best_out,
                                                      float *__restrict__ qnorm, float *__restrict__ qnorm_s,
                                                      CorrOverflow *__restrict__ ovf, unsigned *__restrict__ ovf_count) {
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (q >= g.NQ) return;
    const float *pinb = pin + (size_t)b * g.h * g.w * g.Cp;
    const float *prefb = pref + (size_t)b * g.hr * g.wr * g.Cp;
    const int qp = ((q / g.gw) * g.s_in) * g.w + (q % g.gw) * g.s_in;
    const ImageScale sc = image_scale(sexp, pr_max_bits, rinv_max_bits, g.B, b, is_norm);

    // candidates: slot = CORR_TOPK * chunk + rank; lane l holds slots l, l + 32, l + 64, l + 96 (nchunk <= 32)
    float cv[CORR_TOPK];
    int ci[CORR_TOPK];
    float vmax = -INFINITY;
#pragma unroll
    for (int k = 0; k < CORR_TOPK; ++k) {
        const int slot = lane + 32 * k;
        cv[k] = -INFINITY;
        ci[k] = -1;
        if (slot < CORR_TOPK * nchunk) {
            const Candidate *c = part + ((size_t)b * nchunk + slot / CORR_TOPK) * g.NQ + q;
            cv[k] = c->v[slot % CORR_TOPK];
            ci[k] = c->i[slot % CORR_TOPK];
            if (ci[k] < 0) cv[k] = -INFINITY;
        }
        vmax = fmaxf(vmax, cv[k]);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));

    // A query patch holding NaN / Inf (non-finite in fp64, where no finite fp32 square sum overflows) was searched
    // with those elements read as 0: its lists mean nothing, and all its chunks are re-scanned exactly, always.
    const double qss = query_patch_ss(pinb, g, qp, lane);
    const bool qflag = !isfinite(qss);
    const float qn = (float)sqrt(qss);
    const float qns = (float)ldexp(sqrt(qss), sexp[b]);           // ||P_q|| 2^sexp_in: <= 3 sqrt(C) 1024

    // window = 2E in search units: proportional to ||P_q|| P, the largest |score| the query can have in its image
    // (P = the image's largest ||P_r|| rinv_r), plus the absolute rounding of operand elements that the image's scale exponent leaves in the
    // fp16 subnormals, sub_coef [P + ||P_q|| R], plus the fp32 underflow floor tiny_coef [P + (||P_q|| + 1) R]
    // (c_abi.cu, DESIGN.md K2).  Purely relative to the image's scale: no absolute constant.
    const float floor_u = tiny_coef * (sc.P + (qns + 1.f) * sc.R);
    const float window = window_coef * qns * sc.P + sub_coef * (sc.P + qns * sc.R) + floor_u;
    const float thr = vmax - window;

    // a chunk's list is complete unless something it left behind (`dropped`) reaches the window -> exhaustive re-scan
    unsigned ovf_mask = 0;
    {
        const bool hit = lane < nchunk && (qflag || part[((size_t)b * nchunk + lane) * g.NQ + q].dropped >= thr);
        ovf_mask = __ballot_sync(0xffffffffu, hit);
    }

    // The candidate with the best approximate score is evaluated exactly first (it usually wins); every other in-window
    // candidate first gets the fp32 FMA score and is skipped when even s32 + E32 stays below the best exact score so far.
    const float e32 = e32_coef * qns * sc.P + floor_u;
    const float *rinvb = rinv + (size_t)b * g.NR;
    float best = -INFINITY;
    int besti = 0x7fffffff;
    int first_slot = -1;
    if (!qflag) {
#pragma unroll
        for (int k = 0; k < CORR_TOPK; ++k) {
            const unsigned top = __ballot_sync(0xffffffffu, ci[k] >= 0 && cv[k] == vmax);
            if (first_slot < 0 && top) {
                const int src = __ffs(top) - 1;
                const int r = __shfl_sync(0xffffffffu, ci[k], src);
                const int rp = ((r / g.rw) * g.s_ref) * g.wr + (r % g.rw) * g.s_ref;
                best = exact_score_warp(pinb, prefb, g, qp, rp, is_norm, lane);
                besti = r;
                first_slot = src + 32 * k;
            }
        }
#pragma unroll
        for (int k = 0; k < CORR_TOPK; ++k) {
            unsigned sel = __ballot_sync(0xffffffffu, ci[k] >= 0 && cv[k] >= thr);
            while (sel) {
                const int src = __ffs(sel) - 1;
                sel &= sel - 1;
                if (src + 32 * k == first_slot) continue;                             // done above
                // (listed candidates of a flagged chunk are evaluated too: the re-scan may be skipped by its budget, and
                // then the best LISTED candidate is the result — within 2E of the exact maximum, see corr_rescore_launch)
                const int r = __shfl_sync(0xffffffffu, ci[k], src);
                const int rp = ((r / g.rw) * g.s_ref) * g.wr + (r % g.rw) * g.s_ref;
                // (never against +Inf: an Inf tie goes to the lower index, so it must be scored exactly)
                const float bu = ldexpf(best, sc.u);
                if (bu < INFINITY && fp32_score_warp(pinb, prefb, g, qp, rp, rinvb[r], sc.Sq, sc.Sr, lane) < bu - e32)
                    continue;
                const float s = exact_score_warp(pinb, prefb, g, qp, rp, is_norm, lane);
                if (cand_better(s, r, best, besti)) { best = s; besti = r; }
            }
        }
        // Ref patches holding NaN / Inf never enter the lists (column scale NaN): each is scored exactly here
        const unsigned nflag = flag_count[b];
        for (unsigned i = 0; i < nflag; ++i) {
            const int r = flag_ref[(size_t)b * g.NR + i];
            const int rp = ((r / g.rw) * g.s_ref) * g.wr + (r % g.rw) * g.s_ref;
            const float s = exact_score_warp(pinb, prefb, g, qp, rp, is_norm, lane);
            if (cand_better(s, r, best, besti)) { best = s; besti = r; }
        }
    }
    if (lane == 0) {
        const size_t o = (size_t)b * g.NQ + q;
        best_out[o] = besti == 0x7fffffff ? 0ull : best_key(best, besti);     // 0 sorts below every real key
        qnorm[o] = qn;
        qnorm_s[o] = qns;
        if (qflag) {                                               // from the back: never subject to the budget
            const unsigned n = atomicAdd(ovf_count + 1, 1u);
            ovf[(size_t)g.B * g.NQ - 1 - n] = CorrOverflow{(int)o, ovf_mask};
        } else if (ovf_mask) {
            const unsigned n = atomicAdd(ovf_count, 1u);
            ovf[n] = CorrOverflow{(int)o, ovf_mask};               // capacity B * NQ: one entry per query at most
        }
    }
}

// Exhaustive exact re-scan of the flagged (query, chunk) pairs.  Each list entry is cut into OVF_SPLIT slices of
// the flagged chunks' Ref patches; a block takes (entry, slice) work items grid-stride, its warps stride over the
// slice, and the result is merged into `best` with a 64-bit atomicMax on the packed (score, index) key.
// Per Ref patch a warp first forms the fp32 FMA score (query patch cached in shared memory, ~110 instructions); only
// patches whose fp32 score reaches  (best exact score so far) - E32,  E32 = (K + 8) * 2^-24 * ||P_q|| * ||P_r|| * rinv_r
// (the worst-case error of a K-term fp32 FMA chain; all in search units), can still win and get the exact evaluation
// (~1300 instructions: an IEEE division per element).  With top-4 lists fed by the two best of every 28-patch block
// this runs for a few queries per batch, but it is what makes the candidate lists sufficient instead of "empirically
// enough".  Queries whose patch holds NaN / Inf (entries at the back of the list) are re-scanned without the prefilter
// and whatever the budget.
constexpr int OVF_SPLIT = 64;

__global__ void __launch_bounds__(256) rescore_overflow_kernel(const float *__restrict__ pin, const float *__restrict__ pref,
                                                               const float *__restrict__ rinv, CorrGeom g, CorrChunkGeom cg,
                                                               int nchunk, int is_norm, float e32_coef, float tiny_coef,
                                                               const int *__restrict__ sexp,
                                                               const unsigned *__restrict__ pr_max_bits,
                                                               const unsigned *__restrict__ rinv_max_bits,
                                                               const float *__restrict__ qnorm_s, int qs_floats,
                                                               const CorrOverflow *__restrict__ ovf,
                                                               const unsigned *__restrict__ ovf_count, unsigned budget,
                                                               unsigned long long *__restrict__ best_out) {
    extern __shared__ __align__(16) float qs[];          // scaled query patch [taps][Cp] (qs_floats == 0: no prefilter)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned n_front = ovf_count[0] > budget ? 0u : ovf_count[0];     // tie-flooded input: see corr_rescore_launch
    const unsigned count = n_front + ovf_count[1];
    const int per_tile = cg.tile_rows * cg.tile_cols;
    const int taps = g.patch * g.patch;
    for (unsigned wi = blockIdx.x; wi < count * OVF_SPLIT; wi += gridDim.x) {
        const unsigned e = wi / OVF_SPLIT;
        const CorrOverflow o = e < n_front ? ovf[e] : ovf[(size_t)g.B * g.NQ - 1 - (e - n_front)];
        const int part_i = wi % OVF_SPLIT;
        const int b = o.query / g.NQ, q = o.query - b * g.NQ;
        const float *pinb = pin + (size_t)b * g.h * g.w * g.Cp;
        const float *prefb = pref + (size_t)b * g.hr * g.wr * g.Cp;
        const float *rinvb = rinv + (size_t)b * g.NR;
        const int qp = ((q / g.gw) * g.s_in) * g.w + (q % g.gw) * g.s_in;
        const ImageScale sc = image_scale(sexp, pr_max_bits, rinv_max_bits, g.B, b, is_norm);
        const float qns = qnorm_s[o.query];
        const bool prefilter = qs_floats && isfinite(qns);
        if (prefilter) {
            __syncthreads();                               // previous work item's readers are done
            for (int i = threadIdx.x * 4; i < taps * g.Cp; i += 1024) {
                const int tap = i / g.Cp, c = i - tap * g.Cp;
                float4 v = *reinterpret_cast<const float4 *>(pinb + (size_t)(qp + (tap / g.patch) * g.w + tap % g.patch) * g.Cp + c);
                v.x *= sc.Sq; v.y *= sc.Sq; v.z *= sc.Sq; v.w *= sc.Sq;
                *reinterpret_cast<float4 *>(qs + i) = v;
            }
            __syncthreads();
        }
        float sstar = -INFINITY;                           // exact lower bound on the winner's score, search units
        {
            const unsigned long long k0 = best_out[o.query];
            int r0;
            if (k0 != 0ull) best_unkey(k0, sstar, r0);
            sstar = ldexpf(sstar, sc.u);
        }
        const float e32 = e32_coef * qns * sc.P + tiny_coef * (sc.P + (qns + 1.f) * sc.R);
        float best = -INFINITY;
        int besti = 0x7fffffff;
        for (int c = 0; c < nchunk; ++c) {
            if (!((o.chunks >> c) & 1u)) continue;
            // slots of chunk c: Ref indices (mode 0) or (tile, position) pairs (mode 1); this block's slice of them
            const int n_slots = cg.mode == 0 ? min(g.NR, (c + 1) * cg.per) - c * cg.per
                                             : (min(cg.n_rt, (c + 1) * cg.per) - c * cg.per) * per_tile;
            const int s0 = (int)((long long)n_slots * part_i / OVF_SPLIT), s1 = (int)((long long)n_slots * (part_i + 1) / OVF_SPLIT);
            for (int sl = s0 + warp; sl < s1; sl += 8) {
                int r;
                if (cg.mode == 0) {
                    r = c * cg.per + sl;
                } else {
                    const int rt = c * cg.per + sl / per_tile, w = sl % per_tile;
                    const int ry = (rt / cg.rt_x) * cg.tile_rows + w / cg.tile_cols;
                    const int rx = (rt % cg.rt_x) * cg.tile_cols + w % cg.tile_cols;
                    if (ry >= g.rh || rx >= g.rw) continue;
                    r = ry * g.rw + rx;
                }
                const int rp = ((r / g.rw) * g.s_ref) * g.wr + (r % g.rw) * g.s_ref;
                if (prefilter) {
                    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 3
                    for (int tap = 0; tap < taps; ++tap) {
                        const float *rrow = prefb + (size_t)(rp + (tap / g.patch) * g.wr + tap % g.patch) * g.Cp;
#pragma unroll 2
                        for (int cc = lane * 4; cc < g.Cp; cc += 128) {
                            const float4 rv = *reinterpret_cast<const float4 *>(rrow + cc);
                            const float4 qv = *reinterpret_cast<const float4 *>(qs + tap * g.Cp + cc);
                            a0 = fmaf(qv.x, rv.x * sc.Sr, a0); a1 = fmaf(qv.y, rv.y * sc.Sr, a1);
                            a2 = fmaf(qv.z, rv.z * sc.Sr, a2); a3 = fmaf(qv.w, rv.w * sc.Sr, a3);
                        }
                    }
                    float s32 = (a0 + a1) + (a2 + a3);
#pragma unroll
                    for (int of = 16; of; of >>= 1) s32 += __shfl_xor_sync(0xffffffffu, s32, of);
                    s32 *= rinvb[r];                                         // NaN for a Ref patch holding NaN / Inf
                    // cannot beat the best exact score (warp-uniform); never against +Inf, whose ties go to the lower index
                    const float bu = fmaxf(sstar, ldexpf(best, sc.u));
                    if (bu < INFINITY && s32 < bu - e32) continue;
                }
                const float s = exact_score_warp(pinb, prefb, g, qp, rp, is_norm, lane);
                if (cand_better(s, r, best, besti)) { best = s; besti = r; }
            }
        }
        if (lane == 0 && besti != 0x7fffffff) atomicMax(best_out + o.query, best_key(best, besti));
    }
}

// unpack the winner; val /= ||P_query|| + 1e-5 when norm_input (ref_map_util.py:78-84)
__global__ void __launch_bounds__(256) rescore_finish_kernel(const unsigned long long *__restrict__ best,
                                                             const float *__restrict__ qnorm, int n, int norm_input,
                                                             int64_t *__restrict__ idx, float *__restrict__ val) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n) return;
    const unsigned long long k = best[o];
    float s = -INFINITY;
    int r = 0;
    if (k != 0ull) best_unkey(k, s, r);
    idx[o] = r;
    val[o] = norm_input ? s / (qnorm[o] + 1e-5f) : s;
}

int corr_rescore_launch(const CorrGeom &g, const CorrWorkspace &ws, const CorrChunkGeom &cg, float window_coef,
                        float sub_coef, int is_norm, int norm_input, int64_t *idx, float *val, cudaStream_t st) {
    dim3 grid(ceil_div(g.NQ, 8), g.B);
    const int K = g.Cp * g.patch * g.patch;
    const float e32_coef = ldexpf(1.f, -24) * (float)(K + 8);
    // fp32 underflow floor of both searches and of the prefilters, in search units: a scaled operand element or an
    // fp32 product below 2^-126 rounds by at most 2^-150 (absolute), so a K-term score by (2 K) 2^-150 (||P_r|| rinv_r
    // + ||P_q|| rinv_r + rinv_r); doubled for the window, with margin
    const float tiny_coef = ldexpf(1.f, -146) * (float)(K + 8);
    rescore_kernel<<<grid, 256, 0, st>>>(ws.p32_in, ws.p32_ref, ws.part, g, ws.nchunk, window_coef, sub_coef, e32_coef,
                                         tiny_coef, ws.rinv, ws.pr_max_bits, ws.rinv_max_bits, ws.sexp, is_norm,
                                         ws.flag_ref, ws.flag_count, ws.best, ws.qnorm, ws.qnorm_s, ws.ovf, ws.ovf_count);
    C2M_LAUNCH_CHECK("rescore_kernel");
    // fp32 prefilter of the re-scan: query patch in shared memory when it fits (it does for every model shape)
    const int qs_floats = K * 4 <= 48 * 1024 ? K : 0;
    // Budget of the exhaustive pass.  On inputs whose scores are flooded with near-ties (flat or very smooth images: most
    // Ref patches within the window of most queries) the re-scan degenerates into an exhaustive fp64-exact search — seconds
    // per batch — to order candidates that differ by less than the reference's own fp32 rounding noise.  When more than
    // max(64, queries / 256) queries overflow, the pass is skipped for the whole call (a deterministic, data-only decision)
    // and an overflowed query keeps the exactly-evaluated best of its LISTED candidates.  Every unlisted candidate u of a
    // chunk has s~(u) <= the chunk's listed maximum <= vmax, and the winner w satisfies s(w) >= s(c*) >= vmax - E for
    // the listed candidate c* with s~ = vmax (always evaluated), so s(u) - s(w) <= 2E: the result is within 2E (= the
    // rescoring window) of the exact maximum.  C2M_CORR_EXACT_TIES=1 removes the budget (always exhaustive).  Queries
    // whose patch holds NaN / Inf are outside the budget: they are always re-scanned.
    unsigned budget = (unsigned)(g.B * g.NQ) / 256u;
    if (budget < 64u) budget = 64u;
    if (const char *ev = getenv("C2M_CORR_EXACT_TIES")) if (atoi(ev) != 0) budget = 0xffffffffu;
    rescore_overflow_kernel<<<592, 256, qs_floats * 4, st>>>(ws.p32_in, ws.p32_ref, ws.rinv, g, cg, ws.nchunk, is_norm, e32_coef,
                                                             tiny_coef, ws.sexp, ws.pr_max_bits, ws.rinv_max_bits, ws.qnorm_s,
                                                             qs_floats, ws.ovf, ws.ovf_count, budget, ws.best);
    C2M_LAUNCH_CHECK("rescore_overflow_kernel");
    const int n = g.B * g.NQ;
    rescore_finish_kernel<<<ceil_div(n, 256), 256, 0, st>>>(ws.best, ws.qnorm, n, norm_input, idx, val);
    C2M_LAUNCH_CHECK("rescore_finish_kernel");
    return C2M_OK;
}

}  // namespace c2m
