// Shared pieces of the wgmma implicit-GEMM kernels (plain 3x3 conv, deformable conv):
// parameter blocks and the epilogue that turns one 128-pixel x N-column accumulator (staged in shared
// memory, see acc_store) into packed-split (PSA) and / or strided fp32 output with bias, activation, residuals
// and an optional fused PixelShuffle(2).
#pragma once
#include "c2m_common.cuh"

namespace c2m {

constexpr int UC_NMAX = 64;      // output channels per CTA slice
constexpr int W_HDR = 256;       // packed-weight blob header bytes: [int sw][unsigned bits of max|w|], zero padded

// Weight packing (conv and DCN share the header; their element layouts differ).  Packed weights are split fp16 of
// w * 2^sw.  wpack_header zeroes the header and writes max|w| over the n weights into it (one launch on `st`).
int wpack_header(const float *w, int n, void *packed, cudaStream_t st);
// Grid of a pack kernel (256 threads, grid-stride loop) over `total` packed elements.
inline int wpack_blocks(long long total) { return (int)((total + 255) / 256 > 592 ? 592 : (total + 255) / 256); }

// Prologue of a pack kernel, after wpack_header: sw = 14 - exponent(max|w|), so |w| * 2^sw <= 2^14.  Block 0 writes sw
// to the header for the convolution kernels; returns the scale 2^sw.
__device__ __forceinline__ float wpack_scale(uint8_t *blob) {
    __shared__ int s_sw;
    if (threadIdx.x == 0) {
        const float a = __uint_as_float(reinterpret_cast<unsigned *>(blob)[1]);
        int e = 0;
        if (a > 0.f && isfinite(a)) frexpf(a, &e);
        s_sw = 14 - e;
        if (blockIdx.x == 0) reinterpret_cast<int *>(blob)[0] = s_sw;
    }
    __syncthreads();
    return ldexpf(1.f, s_sw);
}

// Pack loop of a weight blob, after wpack_header: packed element e (fp16, after the header) is the hi or lo half of
// w[src(e, half)] * 2^sw, or 0 where src returns -1 (padding); `src` decodes e and sets `half` (0 hi, 1 lo).  The
// three blob layouts (conv3x3_umma.cu, dcn_umma.cu, dcn_tc_bwd.cu) differ only in that decode.
template <class Src>
__device__ __forceinline__ void wpack_loop(const float *__restrict__ w, uint8_t *blob, long long total, Src src) {
    const float S = wpack_scale(blob);
    __half *dst = reinterpret_cast<__half *>(blob + W_HDR);
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        int half;
        const long long i = src(e, half);
        __half hi, lo;
        psa_split(i >= 0 ? w[i] * S : 0.f, hi, lo);
        dst[e] = half ? lo : hi;
    }
}

// One K chunk (KOCT channel octets, KOCT / 2 K=16 steps) of a 128-row x N tile in split fp16, both operands K-major:
// A = [octet][128 rows][8] per half, octets a_oct bytes apart, rows 64.. starting 1024 B in (acc1); B = [octet][N][8]
// per half.  Three products per step, hi*hi + hi*lo + lo*hi; K chunk kc = 0 starts the accumulators.
template <int N, int KOCT, int R>
__device__ __forceinline__ void wgmma_split_chunk128(float (&acc0)[R], float (&acc1)[R], uint32_t a_hi, uint32_t a_lo,
                                                     uint32_t a_oct, uint32_t w_hi, uint32_t w_lo, int kc) {
    constexpr uint32_t b_lbo = N * 16;
#pragma unroll
    for (int j = 0; j < KOCT / 2; ++j) {
        const uint32_t ao = j * 2 * a_oct, bo = j * 2 * b_lbo;
        const uint64_t dbh = wg_smem_desc(w_hi + bo, b_lbo, 128);
        const uint64_t dbl = wg_smem_desc(w_lo + bo, b_lbo, 128);
        const uint64_t dah = wg_smem_desc(a_hi + ao, a_oct, 128);
        const uint64_t dal = wg_smem_desc(a_lo + ao, a_oct, 128);
        Wgmma<N>::mma(acc0, dah, dbh, (kc | j) != 0);
        Wgmma<N>::mma(acc0, dah, dbl, 1);
        Wgmma<N>::mma(acc0, dal, dbh, 1);
        Wgmma<N>::mma(acc1, wg_desc_advance(dah, 1024), dbh, (kc | j) != 0);
        Wgmma<N>::mma(acc1, wg_desc_advance(dah, 1024), dbl, 1);
        Wgmma<N>::mma(acc1, wg_desc_advance(dal, 1024), dbh, 1);
    }
}

// One K=16 step in split fp16 with both operands MN-major (wgmma_tt_n32): hi*hi + hi*lo + lo*hi into acc
__device__ __forceinline__ void wgmma_tt_split(float (&acc)[16], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi,
                                               uint64_t b_lo) {
    wgmma_tt_n32(acc, a_hi, b_hi);
    wgmma_tt_n32(acc, a_hi, b_lo);
    wgmma_tt_n32(acc, a_lo, b_hi);
}

// Per-image operand exponents of the tensor-core DCN kernels' fp32 boundary (dcn_umma.cu, dcn_tc_bwd.cu), from the bits of the image's largest finite magnitude (0 -> 0).
// x: amax * 2^s in [2^11, 2^12), under fp16's 65504 with 16x headroom for the blend and well above its subnormals.
// mask: max |mask| * 2^s in [1, 2), so the corner weights are at most 2.  Exponent arithmetic only: scaling an image
// by 2^k shifts its exponent by -k and leaves the operand bit for bit the same.  Each exponent is clamped to +-120, so
// 2^sa and 2^sm are normal floats.  Their sum with the weight exponent sw is not clamped: the epilogue's
// 2^-(sa + sm + sw) leaves fp32's range (flushing the output to 0 or overflowing it) only when it exceeds 149 or
// drops below -127.  Since amax(x) 2^sa is in [2^11, 2^12), amax(mask) 2^sm in [1, 2) and amax(w) 2^sw in
// [2^13, 2^14), that happens only when amax(x) amax(mask) amax(w) is below 2^-121 or above 2^151: outputs at the
// edge of fp32's range whatever computes them.
__host__ __device__ __forceinline__ int amax_exp(unsigned bits, int top) {
    if (bits == 0u) return 0;
    const int e = (int)(bits >> 23) - 127;            // floor(log2 amax); a subnormal amax counts as 2^-127
    const int s = top - e;
    return s < -120 ? -120 : s > 120 ? 120 : s;
}
// Per-image exponent of the plain convolution's operands (c2m_conv3x3_operand_f32: x in the forward, grad_output in
// both backwards): sg = 14 - floor(log2 amax) (amax * 2^sg in [2^14, 2^15)), from the bits of the image's largest
// finite |value|; 0 for an all-zero image, clamped to +-120 so that 2^sg and 2^-sg are normal floats.
__host__ __device__ __forceinline__ int grad_scale_exp(const unsigned *amax) { return amax_exp(*amax, 14); }

// ---- Split-K weight gradients (conv3x3_wgrad.cu, dcn_tc_bwd.cu).  dW is a GEMM with M = Cout and K = every pixel of
// the batch.  The pixel tiles are cut into ksplit contiguous K ranges; the CTAs of range k write their fp32 partials
// to workspace slot k, [co_pad][ncol] with column ((c / cpg) * 9 + tap) * cpg + c % cpg holding (channel c, tap): the
// tensor-core DCN's K order, cpg channels per deformable group.  The plain convolution is one group of cpg = ci_pad
// channels, i.e. [co][tap][ci_pad].  wgrad_reduce_kernel sums the slots in one fixed order, so dW is the same bit for
// bit on every run on a given device.

// K ranges of a launch with `ctas` CTAs per range: one wave (the ranges share the SMs), at least one tile per range.
inline int wgrad_ksplit(int ctas, long long ntiles, int &ksplit) {
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    const long long ks = sms / ctas > 0 ? sms / ctas : 1;
    ksplit = (int)(ks < ntiles ? ks : ntiles);
    return C2M_OK;
}

inline size_t wgrad_ws_bytes(int ksplit, int co_pad, int ncol) { return (size_t)ksplit * co_pad * ncol * sizeof(float); }

// Adds the calling warpgroup's NA m64n32 fp32 wgmma accumulators, times 2^e, into a slot and restarts them (`first`
// stores instead of adding).  Accumulator a covers rows [0, 64) x columns [0, 32) from blk + a * stride, row pitch ncol.
// Register i of thread (warp w, lane l) holds row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
// The kernels flush every few tiles because the tensor cores' fp32 accumulation error grows with the number of MMAs
// into one accumulator (linearly, not as a random walk); the slot adds are fp32.
// e sums up to three clamped operand exponents, so 2^e need not be a float: it is one multiply by a normal power of two
// when |e| <= 126 (the common case), else two or three of the same sign.  Each partial product then lies between the
// accumulator and the result, so only the last rounds, as ldexpf would (unless the result is below fp32's normal range).
template <int NA>
__device__ __forceinline__ void wgrad_flush(float (&acc)[NA][16], float *blk, int ncol, int stride, bool first,
                                            int e) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    float *out = blk + (16 * w + (l >> 2)) * ncol + 2 * (l & 3);
    const int e1 = max(-126, min(126, e)), e2 = max(-126, min(126, e - e1));
    const float s1 = ldexpf(1.f, e1), s2 = ldexpf(1.f, e2), s3 = ldexpf(1.f, e - e1 - e2);
    const bool more = e1 != e;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
        float *o0 = out + a * stride, *o1 = o0 + 8 * ncol;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float v = acc[a][i] * s1;
            if (more) v = v * s2 * s3;
            float &d = ((i >> 1) & 1 ? o1 : o0)[8 * (i >> 2) + (i & 1)];
            d = first ? v : d + v;
            acc[a][i] = 0.f;
        }
    }
}

// dW [Cout][C][3][3] = slot 0 + slot 1 + ..., always in that order (the kernels' flushes have divided every operand
// exponent out); one thread per slot column, so the reads
// are coalesced (conv3x3_wgrad.cu; grid-stride over Cout * ncol)
__global__ void wgrad_reduce_kernel(const float *__restrict__ ws, int nslots, int C, int Cout, int cpg, int co_pad,
                                    int ncol, float *__restrict__ dw);

__device__ __forceinline__ int operand_exp(const unsigned *amax, int b) { return amax ? amax_exp(amax[b], 11) : 0; }
__device__ __forceinline__ int mask_exp(const unsigned *amax, int b) { return amax ? amax_exp(amax[b], 0) : 0; }

// fp32 [B,C,H,W] (element strides) -> PSA x * 2^sa, or, when amax is not null, image b times
// 2^grad_scale_exp(amax + b) (conv3x3_umma.cu; grid (blocks, B))
__global__ void psa_from_f32_kernel(const float *__restrict__ x, int C, int C8, int H, int W, long long xs_b,
                                    long long xs_c, long long xs_y, long long xs_x, int sa,
                                    const unsigned *__restrict__ amax, __half *__restrict__ hi,
                                    __half *__restrict__ lo);
// Largest finite |g| of a strided [B,C,H,W] tensor as fp32 bits (NaN and Inf do not set the scale), of the whole batch
// into amax[0] (amax_step 0) or image by image into amax[b] (1); the outputs start at 0 (conv3x3_wgrad.cu; grid
// (blocks, B))
__global__ void grad_amax_kernel(const float *__restrict__ g, int C, int H, int W, long long s_b, long long s_c,
                                 long long s_y, long long s_x, unsigned *__restrict__ amax, int amax_step);

struct ConvParams {
    int B, H, W;
    int nkc_a, nkc;           // K chunks taken from input 1 / in total (input 2 supplies the rest)
    int Cout, N, nslice;      // real couts, couts per CTA slice (multiple of 16), slices; slice s starts at s*N
    int tiles_x, tiles_y;     // 16x8-pixel tiles of one image along x / y
    int act;                  // 0 none, 1 relu, 2 leaky relu 0.1
    int sa_in, sa_res, sa_out;
    int ps;                   // 0 or 2: PixelShuffle(2) applied to the PSA output
    int cs;                   // 1: PSA output stored with st.global.cs (streaming: the DCN output must not evict the
                              // gathered input map from L2)
    int C8out, Hout, Wout;    // geometry of the PSA output tensor
    long long os_b, os_c, os_y, os_x;   // fp32 output element strides
    int f32_mode;             // fp32 output: 0 strided scalar stores, 1 strided with os_c == 1 (16 B stores),
                              // 2 octet-planar [B][ceil(Cout/8)][H][W][8] (two 16 B stores per octet)
};

// fp32 output mode of a strided [B,C,H,W] view: 16 B stores need contiguous channels and aligned strides
inline int f32_store_mode(const float *out, const float *add, long long os_b, long long os_c, long long os_y, long long os_x) {
    const bool al = ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(add)) & 15) == 0;
    return (os_c == 1 && al && os_b % 4 == 0 && os_y % 4 == 0 && os_x % 4 == 0) ? 1 : 0;
}
struct ConvPtrs {
    const uint8_t *wblob;
    const float *bias;
    const __half *res_hi, *res_lo, *res2_hi, *res2_lo;
    __half *out_hi, *out_lo;
    float *out_f32;
    const float *add_f32;
    const unsigned *x_amax;   // [B] or null: image b's input is x * 2^grad_scale_exp(x_amax + b), not x * 2^sa_in
};

// One thread = one output pixel; `acc` points at that pixel's row of the staged accumulator.
// Residual registers of one 32-column block (4 channel octets); fetched by `prefetch_residual`
// BEFORE the thread waits for the accumulator, so the HBM/L2 latency of the residual
// overlaps the MMAs instead of being paid once per octet inside the loop.
struct ResRegs {
    uint4 h[4], l[4];
};

__device__ __forceinline__ void prefetch_residual(const __half *rh, const __half *rl, const ConvParams &p, int b, int y,
                                                  int x, bool ok, int o_base, int c0, ResRegs &r) {
#pragma unroll
    for (int o8 = 0; o8 < 4; ++o8) {
        const int oct = (o_base + c0) / 8 + o8;
        if (ok && c0 + o8 * 8 < p.N && oct < p.C8out) {
            const size_t off = psa_offset(b, oct, y, x, p.C8out, p.H, p.W);
            r.h[o8] = *reinterpret_cast<const uint4 *>(rh + off);
            r.l[o8] = *reinterpret_cast<const uint4 *>(rl + off);
        } else {
            r.h[o8] = make_uint4(0, 0, 0, 0);
            r.l[o8] = make_uint4(0, 0, 0, 0);
        }
    }
}

// One 32-column block [c0, c0+32) of the accumulator.  r1: prefetched first residual (or null);
// a second residual (q.res2_*, rare) is read in place.
__device__ __forceinline__ void epilogue_store_block(const ConvPtrs &q, const ConvParams &p, const float *acc, int c0, int b,
                                                     int y, int x, bool ok, int o_base, const float *sbias,
                                                     float out_scale, float res_scale, float so,
                                                     const ResRegs *r1 = nullptr) {
    uint32_t reg[32];
    acc_ld32(acc, c0, p.N, reg);
    if (!ok) return;
    const int ncol = min(32, p.N - c0);
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        float a = fmaf(__uint_as_float(reg[j]), out_scale, sbias[c0 + j]);
        if (p.act == 1) a = fmaxf(a, 0.f);
        else if (p.act == 2) a = a > 0.f ? a : a * 0.1f;
        v[j] = (j < ncol && o_base + c0 + j < p.Cout) ? a : 0.f;
    }
    if (q.out_f32 && p.f32_mode == 2) {
#pragma unroll
        for (int o8 = 0; o8 < 4; ++o8) {
            const int oct = (o_base + c0) / 8 + o8;
            if (o8 * 8 >= ncol || oct >= p.C8out) break;
            float4 *dst = reinterpret_cast<float4 *>(q.out_f32 + psa_offset(b, oct, y, x, p.C8out, p.H, p.W));
            dst[0] = make_float4(v[o8 * 8], v[o8 * 8 + 1], v[o8 * 8 + 2], v[o8 * 8 + 3]);
            dst[1] = make_float4(v[o8 * 8 + 4], v[o8 * 8 + 5], v[o8 * 8 + 6], v[o8 * 8 + 7]);
        }
    } else if (q.out_f32) {
        const long long base = b * p.os_b + y * p.os_y + x * p.os_x + (long long)(o_base + c0) * p.os_c;
#pragma unroll
        for (int j4 = 0; j4 < 8; ++j4) {
            const int j = j4 * 4, o = o_base + c0 + j;
            if (p.f32_mode == 1 && j + 3 < ncol && o + 3 < p.Cout) {
                float4 val = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                if (q.add_f32) {
                    const float4 ad = *reinterpret_cast<const float4 *>(q.add_f32 + base + j);
                    val.x += ad.x; val.y += ad.y; val.z += ad.z; val.w += ad.w;
                }
                *reinterpret_cast<float4 *>(q.out_f32 + base + j) = val;
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (j + k < ncol && o + k < p.Cout) {
                        const long long oi = base + (j + k) * p.os_c;
                        q.out_f32[oi] = q.add_f32 ? v[j + k] + q.add_f32[oi] : v[j + k];
                    }
            }
        }
    }
    if (q.out_hi && p.ps == 0) {
#pragma unroll
        for (int o8 = 0; o8 < 4; ++o8) {
            const int oct = (o_base + c0) / 8 + o8;
            if (o8 * 8 >= ncol || oct >= p.C8out) break;
            const size_t off = psa_offset(b, oct, y, x, p.C8out, p.H, p.W);
            float r8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (r1) {
#pragma unroll
                for (int j = 0; j < 8; ++j) r8[j] = psa_unsplit(r1->h[o8], r1->l[o8], j) * res_scale;
            }
            if (q.res2_hi) {
                const uint4 rh = *reinterpret_cast<const uint4 *>(q.res2_hi + off);
                const uint4 rl = *reinterpret_cast<const uint4 *>(q.res2_lo + off);
#pragma unroll
                for (int j = 0; j < 8; ++j) r8[j] += psa_unsplit(rh, rl, j) * res_scale;
            }
            __align__(16) __half h8[8];
            __align__(16) __half l8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int o = o_base + c0 + o8 * 8 + j;
                psa_split((o < p.Cout ? v[o8 * 8 + j] + r8[j] : 0.f) * so, h8[j], l8[j]);
            }
            if (p.cs) {
                __stcs(reinterpret_cast<uint4 *>(q.out_hi + off), *reinterpret_cast<const uint4 *>(h8));
                __stcs(reinterpret_cast<uint4 *>(q.out_lo + off), *reinterpret_cast<const uint4 *>(l8));
            } else {
                *reinterpret_cast<uint4 *>(q.out_hi + off) = *reinterpret_cast<const uint4 *>(h8);
                *reinterpret_cast<uint4 *>(q.out_lo + off) = *reinterpret_cast<const uint4 *>(l8);
            }
        }
    }
    if (q.out_hi && p.ps == 2) {
        // PixelShuffle(2): conv channel o = 4c + 2i + j  ->  out[c][2y+i][2x+j]
        // the 32 columns at c0 hold c = (o_base+c0)/4 .. +7  = exactly one output octet
        const int oct = (o_base + c0) / 32;
        if (oct < p.C8out && ncol == 32) {
#pragma unroll
            for (int ij = 0; ij < 4; ++ij) {
                const size_t off = ((((size_t)b * p.C8out + oct) * p.Hout + 2 * y + (ij >> 1)) * p.Wout +
                                    2 * x + (ij & 1)) * 8;
                __align__(16) __half h8[8];
                __align__(16) __half l8[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) psa_split(v[c * 4 + ij] * so, h8[c], l8[c]);
                *reinterpret_cast<uint4 *>(q.out_hi + off) = *reinterpret_cast<const uint4 *>(h8);
                *reinterpret_cast<uint4 *>(q.out_lo + off) = *reinterpret_cast<const uint4 *>(l8);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Specialised epilogue of one full 32-column block (4 complete channel octets): the generic function above spends
// most of its instructions on per-element bounds predicates, activation selects and address arithmetic.  Here
// everything that is uniform per launch is a template parameter and the block is straight-line code.
//   ACT 0 none / 1 ReLU / 2 LeakyReLU(0.1);  RES: one PSA residual (prefetched);  F32OCT: octet-planar fp32 output
//   instead of PSA.
// Preconditions (checked by the caller, warp-uniform): c0 + 32 <= N, o_base + c0 + 32 <= Cout, ps == 0, no res2,
// exactly one output kind.  A PSA output scale 2^sa_out is folded in by the caller: `sbias`, `out_scale` and `res_scale`
// arrive pre-multiplied by it (ReLU / LeakyReLU commute with a positive scale), so it costs nothing per element.
// ---------------------------------------------------------------------------------------------------------------
// Branch-free residual prefetch of a FULL 32-column block (all four octets exist): the loads land directly in their
// final registers.  (The generic prefetch_residual guards every octet with a branch; ptxas then copies each loaded
// value inside its basic block, i.e. waits for one load round trip per octet.)
__device__ __forceinline__ void prefetch_residual_full(const __half *rh, const __half *rl, const ConvParams &p, int b, int y,
                                                       int x, bool ok, int o_base, int c0, ResRegs &r) {
    const size_t plane = (size_t)p.H * p.W * 8;
    const size_t off0 = ((size_t)b * p.C8out + (o_base + c0) / 8) * plane + (ok ? ((size_t)y * p.W + x) * 8 : (size_t)0);
#pragma unroll
    for (int o8 = 0; o8 < 4; ++o8) {
        r.h[o8] = __ldg(reinterpret_cast<const uint4 *>(rh + off0 + o8 * plane));
        r.l[o8] = __ldg(reinterpret_cast<const uint4 *>(rl + off0 + o8 * plane));
    }
}

// The residual octets are fetched BEFORE the thread waits for the accumulator so their HBM / L2 latency overlaps the
// MMAs.  Their fp16 -> fp32 conversion does not depend on the accumulator, so the compiler would hoist it above the
// wait — which puts four serialised load round trips in front of every tile.  This no-op "modifies" the registers
// after the wait, so nothing can consume them earlier.
__device__ __forceinline__ void pin_residual(ResRegs &r) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        asm volatile("" : "+r"(r.h[i].x), "+r"(r.h[i].y), "+r"(r.h[i].z), "+r"(r.h[i].w));
        asm volatile("" : "+r"(r.l[i].x), "+r"(r.l[i].y), "+r"(r.l[i].z), "+r"(r.l[i].w));
    }
}
__device__ __forceinline__ float4 lds_f4(const float *p) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(smem_u32(p)));
    return v;
}

template <int ACT, bool RES, bool F32OCT>
__device__ __forceinline__ void epilogue_fast_block(const ConvPtrs &q, const ConvParams &p, const float *acc, int c0, int b,
                                                    int y, int x, bool ok, int o_base, const float *sbias,
                                                    float out_scale, float res_scale, ResRegs *r1) {
    uint32_t reg[32];
    acc_ld32(acc, c0, c0 + 32, reg);
    if (RES) pin_residual(*r1);
    if (!ok) return;
    const size_t plane = (size_t)p.H * p.W * 8;                       // elements per channel octet
    const size_t off0 = ((size_t)b * p.C8out + (o_base + c0) / 8) * plane + ((size_t)y * p.W + x) * 8;
#pragma unroll
    for (int o8 = 0; o8 < 4; ++o8) {
        const float4 b0 = lds_f4(sbias + c0 + o8 * 8), b1 = lds_f4(sbias + c0 + o8 * 8 + 4);
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float a = fmaf(__uint_as_float(reg[o8 * 8 + j]), out_scale, bb[j]);
            if (ACT == 1) a = fmaxf(a, 0.f);
            else if (ACT == 2) a = fmaxf(a, 0.1f * a);                  // LeakyReLU(0.1): max(a, 0.1 a)
            v[j] = a;
        }
        if (RES) {
            float r[8];
            psa_unsplit2(r1->h[o8], r1->l[o8], r);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = fmaf(r[j], res_scale, v[j]);
        }
        const size_t off = off0 + o8 * plane;
        if (F32OCT) {
            float4 *dst = reinterpret_cast<float4 *>(q.out_f32 + off);
            dst[0] = make_float4(v[0], v[1], v[2], v[3]);
            dst[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
            __align__(16) __half2 h4[4];
            __align__(16) __half2 l4[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) psa_split2(v[2 * j], v[2 * j + 1], h4[j], l4[j]);
            if (p.cs) {
                __stcs(reinterpret_cast<uint4 *>(q.out_hi + off), *reinterpret_cast<const uint4 *>(h4));
                __stcs(reinterpret_cast<uint4 *>(q.out_lo + off), *reinterpret_cast<const uint4 *>(l4));
            } else {
                *reinterpret_cast<uint4 *>(q.out_hi + off) = *reinterpret_cast<const uint4 *>(h4);
                *reinterpret_cast<uint4 *>(q.out_lo + off) = *reinterpret_cast<const uint4 *>(l4);
            }
        }
    }
}

// warp-uniform: can this launch's full blocks take the specialised epilogue?
__device__ __forceinline__ bool epilogue_fast_ok(const ConvPtrs &q, const ConvParams &p) {
    const bool psa_only = q.out_hi && !q.out_f32;
    const bool oct_only = q.out_f32 && p.f32_mode == 2 && !q.out_hi;
    return p.ps == 0 && !q.res2_hi && (psa_only || (oct_only && !q.res_hi && p.sa_out == 0));
}

__device__ __forceinline__ void epilogue_fast_dispatch(const ConvPtrs &q, const ConvParams &p, const float *acc, int c0, int b,
                                                       int y, int x, bool ok, int o_base, const float *sbias,
                                                       float out_scale, float res_scale, ResRegs *r1) {
    const bool oct = q.out_f32 != nullptr;
    if (oct) {
        if (p.act == 0) epilogue_fast_block<0, false, true>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else if (p.act == 1) epilogue_fast_block<1, false, true>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else epilogue_fast_block<2, false, true>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
    } else if (r1) {
        if (p.act == 0) epilogue_fast_block<0, true, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else if (p.act == 1) epilogue_fast_block<1, true, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else epilogue_fast_block<2, true, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
    } else {
        if (p.act == 0) epilogue_fast_block<0, false, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else if (p.act == 1) epilogue_fast_block<1, false, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
        else epilogue_fast_block<2, false, false>(q, p, acc, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, r1);
    }
}

}  // namespace c2m
