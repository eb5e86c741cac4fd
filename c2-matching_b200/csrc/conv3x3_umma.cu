// 3x3 / stride 1 / pad 1 convolution on the sm_90a tensor cores (wgmma) with fp32-grade accuracy
// ("fp16 x 3": split operands hi + lo, hi*hi + hi*lo + lo*hi accumulated in fp32).
//
// SURVEY.md §8(f) N3: once the correlation and DCN are fused, the 128 plain 3x3 convolutions of
// RestorationNet (ResidualBlockNoBN chains, mmsr/models/archs/arch_util.py:80-136;
// ref_restoration_arch.py:22-27,92-95,...) dominate the step when run as exact-fp32 cuDNN
// SIMT kernels.  This kernel keeps fp32-grade results (<= 2^-21 relative per product) at
// tensor-core speed.
//
// Same trick as corr_umma.cu: activations live in the packed-split layout ("PSA")
//      hi, lo : fp16 [B][C/8][H][W][8]
// so ONE TMA box (10 cols x 18 rows x 4 channel octets, origin (x0-1, y0-1): padding = TMA
// out-of-bounds zero fill) per operand half stages a halo'd 16x8-pixel tile in the wgmma
// K-major no-swizzle layout, and the 9 filter taps are MMAs whose A descriptors differ only
// in start address.  The B operand is the weight matrix [Cout x Cin] of the tap, pre-packed
// (c2m_conv3x3_pack_weights_f32) as split fp16 [Cin/32][tap][octet][hi | lo][Cout][8] and kept RESIDENT in
// shared memory for the whole persistent CTA when it fits (<= 147 KB for 64 -> 64), so the only streaming
// traffic is the activation tile.  Epilogue (one output pixel per thread): *2^-(sa+sw) + bias, ReLU /
// LeakyReLU, optional residual add (a second PSA tensor), re-split to hi/lo and store — the
// output is directly the next convolution's operand, no fp32 round trip through HBM.
#include "umma_conv_common.cuh"

namespace c2m {

namespace {
constexpr int T_R = 16, T_C = 8;          // output pixel tile -> M = 128 (two m64 warpgroups)
constexpr int A_R = T_R + 2, A_C = T_C + 2;
constexpr int KOCT = 4;                   // channel octets per K chunk (32 channels)
constexpr int ROW_B = A_C * 16;           // 160 B  (SBO of A)
constexpr int A_OCT_B = A_R * ROW_B;      // 2880 B (LBO of A)
constexpr int A_HALF = KOCT * A_OCT_B;    // 11520 B (hi or lo of one stage)
constexpr int A_STAGE = 2 * A_HALF;       // 23040 B
constexpr int NBST = 2;                   // weight-chunk double buffer
constexpr int NMAX = 64;                  // output channels per CTA slice
// activation ring depth: what is left of the 227 KB next to two weight slots and the accumulator staging
__host__ __device__ constexpr int conv_nstage(int N) { return N >= 64 ? 2 : 4; }
constexpr size_t conv_smem_bytes(int N) {
    return (size_t)NBST * 2 * 9 * KOCT * N * 16 + (size_t)conv_nstage(N) * A_STAGE + acc_stage_bytes(N) + 2048;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// Schedule: CTA c computes the 64-wide Cout slice c % nslice of the 16x8 pixel tiles g = r, r + C, r + 2C, ... of
// the whole batch (tiles numbered image-major, r = c / nslice, C = CTAs per slice).  Tile counts per CTA differ by at
// most one, so no CTA does more than ceil(tiles / C); the CTAs running at any moment sweep neighbouring tiles (their
// halos meet in L2), and the nslice CTAs of one tile are neighbours (they read its activation boxes together).
// Warpgroup 0 produces: warp 0 streams the activation stages (one per (tile, kc), tile-major) through the TMA ring,
// warp 3 bulk-copies the slice's weight chunks (9 taps, hi+lo, N*1152 B per 32-channel chunk kc).  When the chunks
// of a slice fit the two slots (nkc <= 2, i.e. Cin <= 64) they are loaded once per CTA and stay resident; otherwise
// they are streamed per (tile, kc).
// Warpgroups 1 and 2 consume: warpgroup c issues the wgmmas of output rows [64c, 64c + 64) (pixel rows 8c..8c+7)
// of every tile, stages its accumulator in shared memory and runs the epilogue of those 64 pixels.
// Per K step: x_hi * [W_hi | W_lo] (B = the 2N stacked weight rows, n = 2N) + x_lo * W_hi (n = N, into the first
// N columns of the same accumulator); the two halves are summed before staging.
// ------------------------------------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(384, 1)
conv3x3_wgmma_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                     const __grid_constant__ CUtensorMap tm2_hi, const __grid_constant__ CUtensorMap tm2_lo,
                     const ConvPtrs q, const ConvParams p) {
    constexpr int NST = conv_nstage(N);
    constexpr uint32_t w_chunk = 2u * 9 * KOCT * N * 16;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sW = smem;                                                  // [NBST][w_chunk]
    uint8_t *sA = smem + NBST * w_chunk;                                 // multiple of 128 already
    float *acc_s = reinterpret_cast<float *>(sA + NST * A_STAGE);        // [N][ACC_PITCH]
    uint64_t *bars = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(acc_s) + acc_stage_bytes(N));
    uint64_t *full = bars, *empty = full + NST, *bfull = empty + NST, *bempty = bfull + NBST;
    float *sbias = reinterpret_cast<float *>(bempty + NBST);             // [2][UC_NMAX], 16 B aligned (float4 reads)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_img = p.tiles_x * p.tiles_y;
    const int ntiles = p.B * tiles_img;
    // the host launches the same number of CTAs for every slice
    const int slice = blockIdx.x % p.nslice, rank = blockIdx.x / p.nslice, ctas = gridDim.x / p.nslice;
    // global tile index -> (image, top-left output pixel)
    auto tile_at = [&](int g, int &b, int &y0, int &x0) {
        b = g / tiles_img;
        const int tt = g - b * tiles_img;
        y0 = (tt / p.tiles_x) * T_R;
        x0 = (tt % p.tiles_x) * T_C;
    };

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tm_hi);
        tma_prefetch_desc(&tm_lo);
        tma_prefetch_desc(&tm2_hi);
        tma_prefetch_desc(&tm2_lo);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
        for (int i = 0; i < NBST; ++i) { mbar_init(&bfull[i], 1); mbar_init(&bempty[i], 256); }
        fence_mbar_init();
    }
    __syncthreads();
    const int sw = *reinterpret_cast<const int *>(q.wblob);              // weight scale exponent
    // all weight chunks of the slice fit the chunk slots: load them once per CTA, not per tile
    const bool w_resident = p.nkc <= NBST;

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0) {
            // ================================ activation producer ===============================
            if (lane == 0) {
                int stage = 0, phase = 0;
                for (int g = rank; g < ntiles; g += ctas) {
                    int b, y0, x0;
                    tile_at(g, b, y0, x0);
                    for (int kc = 0; kc < p.nkc; ++kc) {
                        const bool first = kc < p.nkc_a;
                        const CUtensorMap *mh = first ? &tm_hi : &tm2_hi, *ml = first ? &tm_lo : &tm2_lo;
                        const int oct0 = (first ? kc : kc - p.nkc_a) * KOCT;
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t *s = sA + stage * A_STAGE;
                        mbar_arrive_expect_tx(&full[stage], A_STAGE);
                        tma_load_4d(s, mh, &full[stage], (x0 - 1) * 8, y0 - 1, oct0, b);
                        tma_load_4d(s + A_HALF, ml, &full[stage], (x0 - 1) * 8, y0 - 1, oct0, b);
                        if (++stage == NST) { stage = 0; phase ^= 1; }
                    }
                }
            }
        } else if (warp == 3) {
            // ================================ weight producer ===================================
            if (lane == 0) {
                int bst = 0, bphase = 0;
                for (int g = rank; g < ntiles; g += ctas) {
                    if (w_resident && g != rank) break;
                    for (int kc = 0; kc < p.nkc; ++kc) {
                        mbar_wait(&bempty[bst], bphase ^ 1);
                        mbar_arrive_expect_tx(&bfull[bst], w_chunk);
                        const uint8_t *src = q.wblob + W_HDR + ((size_t)slice * p.nkc + kc) * w_chunk;
                        for (uint32_t off = 0; off < w_chunk; off += 36864) {
                            const uint32_t n = min(36864u, w_chunk - off);
                            asm volatile(
                                "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                ::"r"(smem_u32(sW + bst * w_chunk + off)), "l"(src + off), "r"(n), "r"(smem_u32(&bfull[bst]))
                                : "memory");
                        }
                        if (++bst == NBST) { bst = 0; bphase ^= 1; }
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ================================ MMA + epilogue ====================================
        const int wg = (warp >> 2) - 1;                      // consumer warpgroup: output rows [64 wg, 64 wg + 64)
        const int wt = threadIdx.x & 127;
        const int e = wg * 64 + (wt & 63);                   // epilogue: pixel of the tile ...
        const int c0 = (wt >> 6) * 32;                       // ... and its 32-column block
        const float out_scale = ldexpf(1.f, -(p.sa_in + sw));
        const float res_scale = ldexpf(1.f, -p.sa_res);
        const float so = ldexpf(1.f, p.sa_out);
        const bool has1 = q.res_hi != nullptr;              // warp-uniform
        const bool fast = epilogue_fast_ok(q, p);           // specialised straight-line epilogue for full blocks
        constexpr uint32_t b_lbo = 2 * N * 16;               // next channel octet of the weights
        constexpr uint32_t a_row0 = 8 * ROW_B;               // the second warpgroup's rows start 8 pixel rows down
        const int o_base = slice * N;
        if (threadIdx.x - 128 < N) {
            const float bv = (q.bias && o_base + (int)threadIdx.x - 128 < p.Cout) ? q.bias[o_base + threadIdx.x - 128] : 0.f;
            sbias[threadIdx.x - 128] = bv;
            sbias[UC_NMAX + threadIdx.x - 128] = bv * so;           // pre-scaled copy for the specialised epilogue
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const bool full_blk = fast && c0 + 32 <= N && o_base + c0 + 32 <= p.Cout;
        int stage = 0, phase = 0, bst = 0, bphase = 0;
        for (int g = rank; g < ntiles; g += ctas) {
            int b, y0, x0;
            tile_at(g, b, y0, x0);
            const int y = y0 + e / T_C, x = x0 + e % T_C;
            const bool ok = y < p.H && x < p.W;
            // per-image input exponents (ops.conv3x3): 2^-(sa_b + sw) for this tile's image.  Past 2^-126 that factor
            // is not a normal float (past 2^-149 it is 0): the accumulator is then first multiplied by 2^-ex, exactly
            // while it stays normal, and the epilogue applies the rest, so an output of ~2^-120 still rounds once.
            const int oe = q.x_amax ? grad_scale_exp(q.x_amax + b) + sw : 0;
            const int ex = oe > 126 ? min(oe - 126, 126) : 0;
            const float osc = q.x_amax ? ldexpf(1.f, ex - oe) : out_scale;
            ResRegs ra;
            if (has1 && c0 < N) {
                if (full_blk) prefetch_residual_full(q.res_hi, q.res_lo, p, b, y, x, ok, o_base, c0, ra);
                else prefetch_residual(q.res_hi, q.res_lo, p, b, y, x, ok, o_base, c0, ra);
            }
            float acc[N];                                        // 64 x 2N: [x*W_hi | x*W_lo] partial sums
            for (int kc = 0; kc < p.nkc; ++kc) {
                const int wslot = w_resident ? kc : bst;         // resident: chunk kc always lives in slot kc
                if (!w_resident || g == rank) mbar_wait(&bfull[wslot], w_resident ? 0 : bphase);
                mbar_wait(&full[stage], phase);
                const uint32_t a_hi = smem_u32(sA + stage * A_STAGE) + wg * a_row0;
                const uint64_t dah = wg_smem_desc(a_hi, A_OCT_B, ROW_B);
                const uint64_t dal = wg_smem_desc(a_hi + A_HALF, A_OCT_B, ROW_B);
                const uint64_t db = wg_smem_desc(smem_u32(sW + wslot * w_chunk), b_lbo, 128);
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
                    for (int j = 0; j < KOCT / 2; ++j) {
                        const uint32_t ao = (tap / 3) * ROW_B + (tap % 3) * 16 + j * 2 * A_OCT_B;
                        const uint32_t bo = (tap * KOCT + j * 2) * b_lbo;
                        Wgmma<2 * N>::mma(acc, wg_desc_advance(dah, ao), wg_desc_advance(db, bo), (kc | tap | j) != 0);
                        Wgmma<N>::mma(acc, wg_desc_advance(dal, ao), wg_desc_advance(db, bo), 1);
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
                mbar_arrive(&empty[stage]);
                if (++stage == NST) { stage = 0; phase ^= 1; }
                if (!w_resident) {
                    mbar_arrive(&bempty[bst]);
                    if (++bst == NBST) { bst = 0; bphase ^= 1; }
                }
            }
            float v[N / 2];
#pragma unroll
            for (int i = 0; i < N / 2; ++i) v[i] = acc[i] + acc[i + N / 2];      // columns c and N + c
            if (ex) {                                                            // uniform per tile
                const float pre = ldexpf(1.f, -ex);
#pragma unroll
                for (int i = 0; i < N / 2; ++i) v[i] *= pre;
            }
            asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");          // previous tile's epilogue is done
            acc_store(acc_s, wg * 64, v);
            asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
            // The residual pointer is a constant in each call: a selected `has1 ? &ra : nullptr` would put `ra` in
            // local memory, and its store there would wait for the prefetch in front of the MMAs.
            if (c0 < N) {
                if (full_blk && has1)
                    epilogue_fast_dispatch(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias + UC_NMAX, osc * so,
                                           res_scale * so, &ra);
                else if (full_blk)
                    epilogue_fast_dispatch(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias + UC_NMAX, osc * so,
                                           res_scale * so, nullptr);
                else if (has1)
                    epilogue_store_block(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias, osc, res_scale, so, &ra);
                else
                    epilogue_store_block(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias, osc, res_scale, so,
                                         nullptr);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// PSA <-> strided fp32 converters and the weight pre-pack
// ------------------------------------------------------------------------------------------
__global__ void psa_from_f32_kernel(const float *__restrict__ x, int C, int C8, int H, int W, long long xs_b,
                                    long long xs_c, long long xs_y, long long xs_x, int sa,
                                    const unsigned *__restrict__ amax, __half *__restrict__ hi,
                                    __half *__restrict__ lo) {
    // one thread = one (octet, pixel); pixel fastest -> coalesced NCHW reads and 16 B stores
    const long long HW = (long long)H * W;
    const long long n = (long long)C8 * HW;
    const int b = blockIdx.y;
    const float S = ldexpf(1.f, amax ? grad_scale_exp(amax + b) : sa);
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int oct = (int)(e / HW);
        const long long pix = e % HW;
        const int y = (int)(pix / W), xx = (int)(pix % W);
        __align__(16) __half h8[8];
        __align__(16) __half l8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = oct * 8 + j;
            psa_split(c < C ? x[b * xs_b + c * xs_c + y * xs_y + xx * xs_x] * S : 0.f, h8[j], l8[j]);
        }
        const size_t o = psa_offset(b, oct, pix, C8, HW);
        *reinterpret_cast<uint4 *>(hi + o) = *reinterpret_cast<const uint4 *>(h8);
        *reinterpret_cast<uint4 *>(lo + o) = *reinterpret_cast<const uint4 *>(l8);
    }
}

__global__ void psa_to_f32_kernel(const __half *__restrict__ hi, const __half *__restrict__ lo, int C, int C8, int H,
                                  int W, int sa, const float *__restrict__ add, float *__restrict__ out, long long os_b,
                                  long long os_c, long long os_y, long long os_x) {
    const long long HW = (long long)H * W;
    const long long n = (long long)C8 * HW;
    const int b = blockIdx.y;
    const float S = ldexpf(1.f, -sa);
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int oct = (int)(e / HW);
        const long long pix = e % HW;
        const int y = (int)(pix / W), xx = (int)(pix % W);
        const size_t o = psa_offset(b, oct, pix, C8, HW);
        const uint4 rh = *reinterpret_cast<const uint4 *>(hi + o);
        const uint4 rl = *reinterpret_cast<const uint4 *>(lo + o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = oct * 8 + j;
            if (c < C) {
                const long long oi = b * os_b + c * os_c + y * os_y + xx * os_x;
                float v = psa_unsplit(rh, rl, j) * S;
                if (add) v += add[oi];
                out[oi] = v;
            }
        }
    }
}

// 2x2 / stride 2 max-pool on a PSA tensor (VGG pool1/pool2 between tensor-core convolutions): the
// pooled map stays in the operand layout, no fp32 round trip through HBM.  max(hi+lo) is taken on
// the reconstructed fp32 values and re-split (the re-split of an already-split value is exact).
__global__ void psa_maxpool2_kernel(const __half *__restrict__ hi, const __half *__restrict__ lo, int C8, int H, int W,
                                    __half *__restrict__ ohi, __half *__restrict__ olo) {
    const int Ho = H / 2, Wo = W / 2;
    const long long n = (long long)C8 * Ho * Wo;
    const int b = blockIdx.y;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int xo = (int)(e % Wo), yo = (int)((e / Wo) % Ho), oct = (int)(e / ((long long)Wo * Ho));
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const size_t o = ((((size_t)b * C8 + oct) * H + 2 * yo + dy) * W + 2 * xo + dx) * 8;
                const uint4 rh = *reinterpret_cast<const uint4 *>(hi + o);
                const uint4 rl = *reinterpret_cast<const uint4 *>(lo + o);
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], psa_unsplit(rh, rl, j));
            }
        __align__(16) __half h8[8];
        __align__(16) __half l8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) psa_split(m[j], h8[j], l8[j]);
        const size_t oo = psa_offset(b, oct, yo, xo, C8, Ho, Wo);
        *reinterpret_cast<uint4 *>(ohi + oo) = *reinterpret_cast<const uint4 *>(h8);
        *reinterpret_cast<uint4 *>(olo + oo) = *reinterpret_cast<const uint4 *>(l8);
    }
}

// blob: [int sw][unsigned amax_bits]...pad to 256 B | [slice][kc][tap][octet][hi|lo][N][8] fp16
// (hi and lo rows of one octet are adjacent: together they are the 2N-row stacked B operand)
__global__ void wpack_kernel(const float *__restrict__ w, int Cin, int Cout, int N, int nkc, int nslice,
                             uint8_t *__restrict__ blob) {
    wpack_loop(w, blob, (long long)nslice * nkc * 2 * 9 * KOCT * N * 8, [=](long long e, int &half) -> long long {
        const int j = (int)(e & 7);
        long long rest = e >> 3;
        const int ol = (int)(rest % N); rest /= N;
        half = (int)(rest % 2); rest /= 2;
        const int oct = (int)(rest % KOCT); rest /= KOCT;
        const int tap = (int)(rest % 9); rest /= 9;
        const int kc = (int)(rest % nkc);
        const int slice = (int)(rest / nkc);
        const int c = (kc * KOCT + oct) * 8 + j, o = slice * NMAX + ol;
        return c < Cin && o < Cout ? ((long long)o * Cin + c) * 9 + tap : -1;
    });
}

int wpack_header(const float *w, int n, void *packed, cudaStream_t st) {
    C2M_CUDA(cudaMemsetAsync(packed, 0, W_HDR, st));
    // the largest FINITE |w|: one Inf weight must not set the scale of all the others (it stays Inf in its own
    // output channel)
    grad_amax_kernel<<<dim3(ceil_div(n, 1024) > 64 ? 64 : ceil_div(n, 1024), 1), 256, 0, st>>>(
        w, 1, 1, n, 0, 0, 0, 1, reinterpret_cast<unsigned *>(packed) + 1, 0);
    C2M_LAUNCH_CHECK("grad_amax_kernel");
    return C2M_OK;
}

// ------------------------------------------------------------------------------------------
static inline int pad16(int c) { return (c + 15) / 16 * 16; }
static inline int n_kc(int cin) { return ((cin + 7) / 8 + KOCT - 1) / KOCT; }
static inline int slice_n(int cout) { return cout <= NMAX ? pad16(cout) : NMAX; }
static inline int n_slice(int cout) { return cout <= NMAX ? 1 : (cout + NMAX - 1) / NMAX; }

}  // namespace c2m

using namespace c2m;

static inline size_t layout1_bytes(int Cin, int Cout) { return (size_t)n_slice(Cout) * n_kc(Cin) * 2 * 9 * KOCT * slice_n(Cout) * 16; }

extern "C" size_t c2m_conv3x3_packed_weight_bytes(int Cin, int Cout) {
    if (Cin <= 0 || Cout <= 0) return 0;
    return (size_t)W_HDR + layout1_bytes(Cin, Cout);
}

extern "C" int c2m_conv3x3_pack_weights_f32(const float *w, int Cin, int Cout, void *packed, c2m_stream_t stream) {
    C2M_CHECK_ARG(w && packed && Cin > 0 && Cout > 0, "conv3x3_pack_weights: bad argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (const int rc = wpack_header(w, Cout * Cin * 9, packed, st)) return rc;
    const int N = slice_n(Cout), nkc = n_kc(Cin), ns = n_slice(Cout);
    const long long total = (long long)ns * nkc * 2 * 9 * KOCT * N * 8;
    wpack_kernel<<<wpack_blocks(total), 256, 0, st>>>(w, Cin, Cout, N, nkc, ns, reinterpret_cast<uint8_t *>(packed));
    C2M_LAUNCH_CHECK("wpack_kernel");
    return C2M_OK;
}

extern "C" int c2m_psa_from_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c,
                                long long xs_y, long long xs_x, int sa, void *hi, void *lo, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && hi && lo && B > 0 && C > 0 && H > 0 && W > 0, "psa_from_f32: bad argument");
    const int C8 = (C + 7) / 8;
    const long long n = (long long)C8 * H * W;
    int bx = (int)((n + 255) / 256);
    if (bx > 4096) bx = 4096;
    psa_from_f32_kernel<<<dim3(bx, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        x, C, C8, H, W, xs_b, xs_c, xs_y, xs_x, sa, nullptr, reinterpret_cast<__half *>(hi),
        reinterpret_cast<__half *>(lo));
    C2M_LAUNCH_CHECK("psa_from_f32_kernel");
    return C2M_OK;
}

extern "C" int c2m_psa_to_f32(const void *hi, const void *lo, int B, int C, int H, int W, int sa, const float *add,
                              float *out, long long os_b, long long os_c, long long os_y, long long os_x,
                              c2m_stream_t stream) {
    C2M_CHECK_ARG(out && hi && lo && B > 0 && C > 0 && H > 0 && W > 0, "psa_to_f32: bad argument");
    const int C8 = (C + 7) / 8;
    const long long n = (long long)C8 * H * W;
    int bx = (int)((n + 255) / 256);
    if (bx > 4096) bx = 4096;
    psa_to_f32_kernel<<<dim3(bx, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half *>(hi), reinterpret_cast<const __half *>(lo), C, C8, H, W, sa, add, out, os_b,
        os_c, os_y, os_x);
    C2M_LAUNCH_CHECK("psa_to_f32_kernel");
    return C2M_OK;
}

extern "C" int c2m_psa_maxpool2(const void *hi, const void *lo, int B, int C, int H, int W, void *out_hi, void *out_lo,
                                c2m_stream_t stream) {
    C2M_CHECK_ARG(hi && lo && out_hi && out_lo && B > 0 && C > 0 && H >= 2 && W >= 2, "psa_maxpool2: bad argument");
    const int C8 = (C + 7) / 8;
    const long long n = (long long)C8 * (H / 2) * (W / 2);
    int bx = (int)((n + 255) / 256);
    if (bx > 4096) bx = 4096;
    psa_maxpool2_kernel<<<dim3(bx, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half *>(hi), reinterpret_cast<const __half *>(lo), C8, H, W,
        reinterpret_cast<__half *>(out_hi), reinterpret_cast<__half *>(out_lo));
    C2M_LAUNCH_CHECK("psa_maxpool2_kernel");
    return C2M_OK;
}

extern "C" int c2m_conv3x3(const c2m_conv3x3_args *a, c2m_stream_t stream) {
    C2M_CHECK_ARG(a, "conv3x3: null args");
    C2M_CHECK_ARG(a->in_hi && a->in_lo && a->packed_w, "conv3x3: null input / weights");
    C2M_CHECK_ARG(a->B > 0 && a->Cin > 0 && a->Cout > 0, "conv3x3: bad shape");
    C2M_CHECK_ARG(a->H >= A_R && a->W >= A_C, "conv3x3: map %dx%d smaller than one halo tile (18x10)", a->H, a->W);
    C2M_CHECK_ARG((a->in2_hi == nullptr) == (a->Cin2 == 0) && (a->in2_hi == nullptr) == (a->in2_lo == nullptr),
                  "conv3x3: inconsistent second input");
    C2M_CHECK_ARG(a->Cin2 == 0 || a->Cin % (KOCT * 8) == 0,
                  "conv3x3: first of two concatenated inputs must have a multiple of 32 channels (got %d)", a->Cin);
    C2M_CHECK_ARG((a->res_hi == nullptr) == (a->res_lo == nullptr) && (a->res2_hi == nullptr) == (a->res2_lo == nullptr),
                  "conv3x3: residual needs both halves");
    C2M_CHECK_ARG(a->act >= 0 && a->act <= 2, "conv3x3: unknown activation %d", a->act);
    C2M_CHECK_ARG(!a->x_amax || !a->in2_hi, "conv3x3: per-image input exponents need a single input");
    C2M_CHECK_ARG((a->out_hi == nullptr) == (a->out_lo == nullptr), "conv3x3: PSA output needs both halves");
    C2M_CHECK_ARG(a->out_hi || a->out_f32, "conv3x3: no output requested");
    C2M_CHECK_ARG(a->pixel_shuffle == 0 || (a->pixel_shuffle == 2 && a->Cout % 32 == 0 && a->out_hi && !a->res_hi),
                  "conv3x3: pixel_shuffle must be 0 or 2 (Cout %% 32 == 0, PSA output, no residual)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    ConvParams p;
    p.B = a->B; p.H = a->H; p.W = a->W;
    p.nkc_a = n_kc(a->Cin);
    p.nkc = a->Cin2 ? a->Cin / (KOCT * 8) + n_kc(a->Cin2) : p.nkc_a;
    if (a->Cin2) p.nkc_a = a->Cin / (KOCT * 8);
    p.Cout = a->Cout; p.N = slice_n(a->Cout); p.nslice = n_slice(a->Cout);
    p.tiles_x = ceil_div(a->W, T_C); p.tiles_y = ceil_div(a->H, T_R);
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    p.cs = 0;
    p.act = a->act; p.sa_in = a->sa_in; p.sa_res = a->sa_res; p.sa_out = a->sa_out;
    p.ps = a->pixel_shuffle;
    const int c_out_psa = p.ps == 2 ? a->Cout / 4 : a->Cout;
    p.C8out = (c_out_psa + 7) / 8;
    p.Hout = p.ps == 2 ? 2 * a->H : a->H;
    p.Wout = p.ps == 2 ? 2 * a->W : a->W;
    p.os_b = a->os_b; p.os_c = a->os_c; p.os_y = a->os_y; p.os_x = a->os_x;
    C2M_CHECK_ARG(!a->out_f32_octets || (a->out_f32 && !a->add_f32 && (reinterpret_cast<uintptr_t>(a->out_f32) & 15) == 0),
                  "conv3x3: octet-planar fp32 output needs a 16 B aligned out_f32 and no add_f32");
    p.f32_mode = !a->out_f32 ? 0 : a->out_f32_octets ? 2 : f32_store_mode(a->out_f32, a->add_f32, a->os_b, a->os_c, a->os_y, a->os_x);
    ConvPtrs q;
    q.wblob = reinterpret_cast<const uint8_t *>(a->packed_w);
    q.bias = a->bias;
    q.res_hi = reinterpret_cast<const __half *>(a->res_hi); q.res_lo = reinterpret_cast<const __half *>(a->res_lo);
    q.res2_hi = reinterpret_cast<const __half *>(a->res2_hi); q.res2_lo = reinterpret_cast<const __half *>(a->res2_lo);
    q.out_hi = reinterpret_cast<__half *>(a->out_hi); q.out_lo = reinterpret_cast<__half *>(a->out_lo);
    q.out_f32 = a->out_f32; q.add_f32 = a->add_f32;
    q.x_amax = a->x_amax;
    CUtensorMap mh, ml, m2h, m2l;
    int rc;
    if ((rc = make_psa_tensor_map(&mh, a->in_hi, a->B, (a->Cin + 7) / 8, a->H, a->W, A_C, A_R))) return rc;
    if ((rc = make_psa_tensor_map(&ml, a->in_lo, a->B, (a->Cin + 7) / 8, a->H, a->W, A_C, A_R))) return rc;
    if (a->Cin2) {
        if ((rc = make_psa_tensor_map(&m2h, a->in2_hi, a->B, (a->Cin2 + 7) / 8, a->H, a->W, A_C, A_R))) return rc;
        if ((rc = make_psa_tensor_map(&m2l, a->in2_lo, a->B, (a->Cin2 + 7) / 8, a->H, a->W, A_C, A_R))) return rc;
    } else {
        m2h = mh; m2l = ml;
    }
    C2M_CUDA(cudaFuncSetAttribute(conv3x3_wgmma_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)conv_smem_bytes(16)));
    C2M_CUDA(cudaFuncSetAttribute(conv3x3_wgmma_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)conv_smem_bytes(32)));
    C2M_CUDA(cudaFuncSetAttribute(conv3x3_wgmma_kernel<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)conv_smem_bytes(48)));
    C2M_CUDA(cudaFuncSetAttribute(conv3x3_wgmma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)conv_smem_bytes(64)));
    // one persistent CTA per SM, the same number for every slice, and no more per slice than there are tiles
    const int tiles = a->B * p.tiles_x * p.tiles_y;
    const int fit = sms / p.nslice > 0 ? sms / p.nslice : 1;
    const int grid = p.nslice * (tiles < fit ? tiles : fit);
    // algorithmic work: 2*Cin*Cout*9 flops per output pixel; bytes = PSA in (4 B/elem) + out
    const double cin_t = (double)a->Cin + a->Cin2, px = (double)a->B * a->H * a->W;
    const double flops = 2.0 * cin_t * a->Cout * 9.0 * px;
    const double bytes = 4.0 * px * (cin_t + a->Cout * ((a->out_hi ? 1 : 0) + (a->out_f32 ? 1 : 0)) +
                                     a->Cout * ((a->res_hi ? 1 : 0) + (a->res2_hi ? 1 : 0) + (a->add_f32 ? 1 : 0)));
    void *ph = prof_begin(PROF_CONV3X3, flops, bytes, st);
    switch (p.N) {
    case 16: conv3x3_wgmma_kernel<16><<<grid, 384, conv_smem_bytes(16), st>>>(mh, ml, m2h, m2l, q, p); break;
    case 32: conv3x3_wgmma_kernel<32><<<grid, 384, conv_smem_bytes(32), st>>>(mh, ml, m2h, m2l, q, p); break;
    case 48: conv3x3_wgmma_kernel<48><<<grid, 384, conv_smem_bytes(48), st>>>(mh, ml, m2h, m2l, q, p); break;
    default: conv3x3_wgmma_kernel<64><<<grid, 384, conv_smem_bytes(64), st>>>(mh, ml, m2h, m2l, q, p); break;
    }
    C2M_LAUNCH_CHECK("conv3x3_wgmma_kernel");
    prof_end(ph, st);
    return C2M_OK;
}
