// Shared helpers for libc2m_sm100: error plumbing, launch accounting and the sm_90a PTX
// wrappers (mbarrier, TMA, wgmma) used by the kernels.  sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/c2m_sm100.h"
#include "wgmma_f16.cuh"

namespace c2m {

// ---------------------------------------------------------------------------- host side
void set_error(const char *fmt, ...);
void count_launch(unsigned n = 1);

// Measurement hook (include/c2m_sm100.h c2m_profile_*): kernel classes timed with CUDA events on the
// launching stream while profiling is enabled.
enum ProfKernel { PROF_CORR_SEARCH = 0, PROF_CONV3X3 = 1, PROF_DCN = 2, PROF_DCN_DGRAD = 3, PROF_DCN_WGRAD = 4,
                  PROF_CONV3X3_WGRAD = 5, PROF_NKERNELS = 6 };
bool prof_enabled();
void *prof_begin(int kernel, double flops, double bytes, cudaStream_t st);   // null when disabled
void prof_end(void *handle, cudaStream_t st);

#define C2M_CHECK_ARG(cond, ...)                 \
    do {                                         \
        if (!(cond)) {                           \
            c2m::set_error(__VA_ARGS__);         \
            return C2M_ERR_INVALID;              \
        }                                        \
    } while (0)

#define C2M_CUDA(call)                                                                        \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            c2m::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, \
                           __LINE__);                                                         \
            return C2M_ERR_CUDA;                                                              \
        }                                                                                     \
    } while (0)

#define C2M_LAUNCH_CHECK(name)                                                         \
    do {                                                                               \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) {                                                      \
            c2m::set_error("launch of %s failed: %s", name, cudaGetErrorString(e__)); \
            return C2M_ERR_CUDA;                                                       \
        }                                                                              \
        c2m::count_launch();                                                           \
    } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
__host__ __device__ static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Blocks of 256 threads for a grid-stride loop over n items: one per 256 items, at most 16 per SM of an H100.
static inline int grid_blocks(long long n) {
    const long long b = (n + 255) / 256;
    return (int)(b < 132 * 16 ? b : 132 * 16);
}

// number of SMs of the current device (the persistent kernels launch at most one CTA per SM)
static inline cudaError_t sm_count(int &sms) {
    int dev = 0;
    const cudaError_t e = cudaGetDevice(&dev);
    return e != cudaSuccess ? e : cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
}

// TMA descriptor of a PSA half-plane fp16 [B][C8][H][W][8] as the 4-D tensor (W*8, H, C8, B); one box is
// box_px pixels x box_rows rows x 4 channel octets of one image.  Out-of-bounds elements load as zero.
int make_psa_tensor_map(CUtensorMap *map, const void *base, int B, int C8, int H, int W, int box_px, int box_rows);

// ---------------------------------------------------------------------------- device side
#ifdef __CUDACC__
// max |x[i]| over n floats, folded into *out_bits (float bits, start at 0); corr_aux.cu
__global__ void amax_kernel(const float *__restrict__ x, size_t n, unsigned *__restrict__ out_bits);

// ---- packed-split (PSA) format: every tensor-core operand and PSA activation.  A value v is the fp16 pair
// hi = rn(v), lo = rn(v - hi) (|lo| <= 2^-11 |v|, so hi + lo carries ~22 bits of v), and a product of two such values
// is the three MMAs hi*hi + hi*lo + lo*hi (the correlation search drops the Ref's lo, corr_umma.cu).  A tensor
// [B][C][H][W] is stored as two fp16 planes (hi, lo), each laid out as channel octets [B][ceil(C/8)][H][W][8] with the
// padding channels of the last octet zero; the tensor-core DCN's operand interleaves them per octet, [hi 8 | lo 8].
// The split and the unsplit come in a per-element (__half) and a per-pair (__half2) form; each site keeps the form it
// was tuned with (they round alike but compile differently).
__device__ __forceinline__ void psa_split(float v, __half &hi, __half &lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}
__device__ __forceinline__ void psa_split2(float a, float b, __half2 &hi, __half2 &lo) {
    hi = __floats2half2_rn(a, b);
    const float2 f = __half22float2(hi);
    lo = __floats2half2_rn(a - f.x, b - f.y);
}
// hi + lo of one octet (16 B of each half): element j, or all 8 converted pairwise
__device__ __forceinline__ float psa_unsplit(const uint4 &hi, const uint4 &lo, int j) {
    return __half2float(reinterpret_cast<const __half *>(&hi)[j]) + __half2float(reinterpret_cast<const __half *>(&lo)[j]);
}
__device__ __forceinline__ void psa_unsplit2(const uint4 &hi, const uint4 &lo, float (&v)[8]) {
    const __half2 *h = reinterpret_cast<const __half2 *>(&hi), *l = reinterpret_cast<const __half2 *>(&lo);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(h[j]), b = __half22float2(l[j]);
        v[2 * j] = a.x + b.x;
        v[2 * j + 1] = a.y + b.y;
    }
}
// element offset of octet `oct` of pixel (y, x) of image b in one half-plane; the second form takes the pixel index
// pix = y * W + x of an HW = H * W plane
__device__ __forceinline__ size_t psa_offset(int b, int oct, int y, int x, int C8, int H, int W) {
    return ((((size_t)b * C8 + oct) * H + y) * W + x) * 8;
}
__device__ __forceinline__ size_t psa_offset(int b, int oct, long long pix, int C8, long long HW) {
    return (((size_t)b * C8 + oct) * HW + pix) * 8;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug (lost arrive, register-pool deadlock, ...) must end in a trap that the
// host sees as a launch failure, not in a kernel that spins until the GPU lease is killed.  One try_wait
// probe suspends for up to ~1 us, so the limit below is tens of seconds; -DC2M_MBAR_SPIN_LIMIT=0 removes
// the counter.
#ifndef C2M_MBAR_SPIN_LIMIT
#define C2M_MBAR_SPIN_LIMIT (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
#if C2M_MBAR_SPIN_LIMIT
    uint32_t n = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++n > C2M_MBAR_SPIN_LIMIT) __trap();   // no printf here: it would put a stack frame into every role loop
    }
#else
    while (!mbar_try_wait(bar, parity)) {
    }
#endif
}
// (A hinted variant — try_wait with a suspend-time hint, which compiles to NANOSLEEP.SYNCS — was measured
// for the long epilogue / producer waits: no change in step time or power, so the plain probe loop stays.)

// ---- TMA (cp.async.bulk.tensor), 4-D tiled load into this CTA's shared memory
__device__ __forceinline__ void tma_prefetch_desc(const void *tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void *dst, const void *tmap, uint64_t *bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---- wgmma (warpgroup MMA, sm_90a): issued by all 128 threads of a warpgroup, accumulator in registers
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Shared-memory matrix descriptor, K-major, no swizzle ("interleave"): core matrix = 8 rows x 16 bytes, rows 16 B
// apart; `lbo` = byte distance between the two K core matrices of one K=16 step, `sbo` = byte distance between
// consecutive 8-row groups along M/N.  Fields: start[0,14) lbo[16,30) sbo[32,46), layout type [62,64) = 0.
__device__ __forceinline__ uint64_t wg_smem_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
// Same descriptor advanced by `byte_off` (multiple of 16; the 14-bit start-address field cannot carry: shared
// memory is < 2^18 bytes) — one 32-bit add on the low word.
__device__ __forceinline__ uint64_t wg_desc_advance(uint64_t desc, uint32_t byte_off) {
    const uint32_t lo = (uint32_t)desc + (byte_off >> 4);
    return (desc & 0xFFFFFFFF00000000ull) | lo;
}

// ---- accumulator staging: the epilogues read a finished tile from shared memory as [column][row] fp32 with
// ACC_PITCH floats per column (row fastest: one thread per row reads a column without bank conflicts, and the
// fragment stores below hit 32 distinct banks because 2 * ACC_PITCH = 8 mod 32).
constexpr int ACC_PITCH = 132;
__host__ __device__ constexpr int acc_stage_bytes(int cols) { return cols * ACC_PITCH * 4; }

// Store the calling warpgroup's 64 x (2R) wgmma fragment as rows [row0, row0 + 64) of the staging buffer.
template <int R>
__device__ __forceinline__ void acc_store(float *acc_s, int row0, const float (&d)[R]) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    float *base = acc_s + row0 + 16 * w + (l >> 2) + 2 * (l & 3) * ACC_PITCH;
#pragma unroll
    for (int i = 0; i < R; ++i) base[(8 * (i >> 2) + (i & 1)) * ACC_PITCH + 8 * ((i >> 1) & 1)] = d[i];
}
// Columns [c0, c0 + 32) of one row (`acc_row` = staging buffer + row); columns at or beyond `ncol` read as 0.
__device__ __forceinline__ void acc_ld32(const float *acc_row, int c0, int ncol, uint32_t (&r)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) r[j] = c0 + j < ncol ? __float_as_uint(acc_row[(c0 + j) * ACC_PITCH]) : 0u;
}
#endif  // __CUDACC__

}  // namespace c2m
