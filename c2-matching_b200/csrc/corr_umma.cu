// Fused all-pairs patch correlation + running top-k on the sm_90a tensor cores (wgmma).
//
// Replaces the reference's chunked `F.conv2d(feat_in, ref_patches)` + `max`
// (mmsr/models/archs/ref_map_util.py:54-76), which materialises a [n_ref, h', w'] score tensor
// per chunk (2 x 2.09 GB per image at 160x160 maps).  Here no score ever reaches HBM.
//
// Formulation.  score(q,r) = sum_{dy,dx in 3x3} sum_c in[q+(dy,dx)][c] * ref[r+(dy,dx)][c].  The row taps go to
// the tensor core, the column taps to the epilogue:
//     V(p, s)     = sum_{dy} sum_c in[p+(dy,0)][c] * ref[s+(dy,0)][c]          GEMM, K = 3*C (a third of 9*C)
//     score(q, r) = V(q, r) + V(q+(0,1), r+(0,1)) + V(q+(0,2), r+(0,2))        3-term diagonal sum
// Pixel blocks are 16 columns wide on both sides (14 patch origins + 2 halo columns), stored by ONE TMA box per
// operand half as [octet][row][16 px][8 halfs]: 16 px x 16 B = 256 B rows are contiguous, so M index m = 16*row + x
// (query block: 8 rows -> M = 128) and N index n = 16*row + x (Ref block: 8 rows -> N = 128) are CONTIGUOUS pixel
// runs in the wgmma K-major no-swizzle layout (8-pixel core-matrix groups 128 B apart = SBO, channel octets
// one block apart = LBO), and the row tap dy is a +256 B start-address offset on both descriptors.
// In the staged accumulator, row m+dx / column n+dx hold V(q+(0,dx), r+(0,dx)); the epilogue runs one thread per
// row, so a warp's 32 threads are exactly two 16-px block rows and the diagonal sum is two __shfl_down per score.
// Tile efficiency (14/16)^2 = 0.77, i.e. 2.3x fewer MMA cycles per score than issuing all nine taps.
//
// Precision.  Operands are split fp16 pairs of x*2^sexp[b] (hi + lo, 22 mantissa bits); each K step
// issues q_hi*r_hi + q_lo*r_hi into the same fp32 accumulator (M=128, N=128).  The scores
// only RANK candidates: the epilogue keeps a top-8 per (query, Ref chunk) and the exact rescoring kernel
// (corr_aux.cu) decides, so tensor-core rounding cannot leak into the index map; corr_aux.cu states the error
// bound that sizes the rescoring window and the exhaustive fallback that makes the top-8 lists sufficient.
//
// CTA = 512 threads: warp 0 TMA producer, warps 4-7 epilogue (one accumulator row per thread), warps 8-15 two
// MMA warpgroups (accumulator rows 0-63 / 64-127, 64 fp32 registers per thread).  4-stage smem ring (30 KB per
// stage); a finished accumulator is staged in shared memory, so the epilogue of Ref tile n overlaps the MMAs of
// tile n+1 (which accumulate in registers).  Persistent: grid = #SMs, work item = (image, query tile, Ref chunk).
#include "corr_internal.cuh"

namespace c2m {

namespace {
constexpr int PATCH = 3;
constexpr int BW = 16;                             // block width in pixels (both sides)
constexpr int TV = BW - (PATCH - 1);               // 14 valid patch origins per block row
constexpr int TQ_R = 8;                            // query block rows  -> M = 8 * 16 = 128 (two m64 warpgroups)
constexpr int TR_R = 8;                            // Ref block rows    -> wgmma N = 8 * 16 = 128
constexpr int A_R = TQ_R + PATCH - 1;              // 10 staged rows
constexpr int B_R = TR_R + PATCH - 1;              // 10
constexpr int KOCT = 4;                            // channel octets per stage (32 channels)
constexpr int ROW_B = BW * 16;                     // 256 B block row pitch (= row-tap offset)
constexpr int A_OCT_B = A_R * ROW_B;               // 2560 B octet pitch of A (= LBO)
constexpr int B_OCT_B = B_R * ROW_B;               // 2560 B octet pitch of B (= LBO)
constexpr int A_BYTES = KOCT * A_OCT_B;            // 10240
constexpr int B_BYTES = KOCT * B_OCT_B;            // 10240
constexpr int STAGE_BYTES = 2 * A_BYTES + B_BYTES;     // query hi + lo, Ref hi = 30720
constexpr int NSTAGE = 4;
constexpr int UM = TQ_R * BW, UN = TR_R * BW;      // 128, 128
constexpr int SMEM_AUX = 2 * UN * 8 + 128;         // (scale, bias) per column, double buffered, + barriers
constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + acc_stage_bytes(UN) + SMEM_AUX + 1024;
static_assert(A_BYTES % 128 == 0 && B_BYTES % 128 == 0, "TMA destinations must stay 128B aligned");
static_assert(UM == 128 && UN == 128, "tile shape: two m64 warpgroups x an n128 wgmma");
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");

struct UmmaParams {
    int B, C8;
    int gh, gw, rh, rw;          // patch grids
    int qt_x, qt_y, rt_x, rt_y;  // tile counts
    int nchunk, rt_per_chunk;
    int NQ, NR;
};
}  // namespace

__global__ void __launch_bounds__(512, 1)
corr_umma_kernel(const __grid_constant__ CUtensorMap tm_in_hi, const __grid_constant__ CUtensorMap tm_in_lo,
                 const __grid_constant__ CUtensorMap tm_ref_hi,
                 const float *__restrict__ rinv, Candidate *__restrict__ part,
                 const UmmaParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float *acc_s = reinterpret_cast<float *>(smem + NSTAGE * STAGE_BYTES);          // [UN][ACC_PITCH]
    uint8_t *aux = smem + NSTAGE * STAGE_BYTES + acc_stage_bytes(UN);
    float2 *rcol = reinterpret_cast<float2 *>(aux);                 // [2][UN] (score scale, bias)
    uint64_t *bars = reinterpret_cast<uint64_t *>(aux + 2 * UN * 8);
    uint64_t *full = bars, *empty = bars + NSTAGE, *tfull = bars + 2 * NSTAGE, *tempty = bars + 2 * NSTAGE + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tm_in_hi);
        tma_prefetch_desc(&tm_in_lo);
        tma_prefetch_desc(&tm_ref_hi);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NSTAGE; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
        mbar_init(tfull, 256);
        mbar_init(tempty, 4);
        fence_mbar_init();
    }
    __syncthreads();

    const int n_qt = p.qt_x * p.qt_y, n_rt = p.rt_x * p.rt_y;
    const int n_items = p.B * n_qt * p.nchunk;
    const int n_kc = (p.C8 + KOCT - 1) / KOCT;

    if (warp < 4) {
        // ================================ TMA producer =====================================
        if (warp == 0 && lane == 0) {
            int stage = 0, phase = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int chunk = item % p.nchunk, qt = (item / p.nchunk) % n_qt, b = item / (p.nchunk * n_qt);
                const int qy0 = (qt / p.qt_x) * TQ_R, qx0 = (qt % p.qt_x) * TV;
                const int rt_b = chunk * p.rt_per_chunk, rt_e = min(n_rt, rt_b + p.rt_per_chunk);
                for (int rt = rt_b; rt < rt_e; ++rt) {
                    const int ry0 = (rt / p.rt_x) * TR_R, rx0 = (rt % p.rt_x) * TV;
                    for (int kc = 0; kc < n_kc; ++kc) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t *s = smem + stage * STAGE_BYTES;
                        mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
                        tma_load_4d(s, &tm_in_hi, &full[stage], qx0 * 8, qy0, kc * KOCT, b);
                        tma_load_4d(s + A_BYTES, &tm_in_lo, &full[stage], qx0 * 8, qy0, kc * KOCT, b);
                        tma_load_4d(s + 2 * A_BYTES, &tm_ref_hi, &full[stage], rx0 * 8, ry0, kc * KOCT, b);
                        if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else if (warp >= 8) {
        // ================================ MMA ==============================================
        // warpgroup wg computes accumulator rows [64 wg, 64 wg + 64) (query block rows 4 wg .. 4 wg + 3): its A
        // operand starts 8 core-matrix groups (1024 B) further in
        const int wg = (warp >> 2) - 2;
        int stage = 0, phase = 0;
        uint32_t tphase = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int chunk = item % p.nchunk;
            const int rt_b = chunk * p.rt_per_chunk, rt_e = min(n_rt, rt_b + p.rt_per_chunk);
            for (int rt = rt_b; rt < rt_e; ++rt) {
                float acc[UN / 2];
                for (int kc = 0; kc < n_kc; ++kc) {
                    mbar_wait(&full[stage], phase);
                    const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
                    // descriptors of (row tap 0, k-step 0); every other MMA is a constant offset away
                    const uint64_t dah0 = wg_smem_desc(sa + wg * 1024, A_OCT_B, 128);
                    const uint64_t dal0 = wg_smem_desc(sa + A_BYTES + wg * 1024, A_OCT_B, 128);
                    const uint64_t dbh0 = wg_smem_desc(sa + 2 * A_BYTES, B_OCT_B, 128);
                    wgmma_fence();
#pragma unroll
                    for (int dy = 0; dy < PATCH; ++dy) {
#pragma unroll
                        for (int j = 0; j < KOCT / 2; ++j) {
                            const uint32_t ao = dy * ROW_B + j * 2 * A_OCT_B, bo = dy * ROW_B + j * 2 * B_OCT_B;
                            const uint64_t dbh = wg_desc_advance(dbh0, bo);
                            // (q_hi + q_lo) * r_hi: the query keeps its 22-bit split, the Ref operand is its fp16
                            // rounding.  The search only RANKS; the 2^-11 this costs is part of the rescoring
                            // window (DESIGN.md K2).
                            Wgmma<UN>::mma(acc, wg_desc_advance(dah0, ao), dbh, (kc | dy | j) != 0);
                            Wgmma<UN>::mma(acc, wg_desc_advance(dal0, ao), dbh, 1);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait_all();
                    mbar_arrive(&empty[stage]);                 // smem slot free
                    if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
                }
                mbar_wait(tempty, tphase ^ 1);                  // the epilogue has read the previous tile
                acc_store(acc_s, wg * 64, acc);
                mbar_arrive(tfull);                             // accumulator complete
                tphase ^= 1;
            }
        }
    } else {
        // ================================ epilogue =========================================
        // Branch-free inner loop: per 32-column block (two Ref block rows, 28 valid scores) only min / max run per
        // score — m1 >= m2 >= m3 = the block's three best — and only m1, m2 are offered to the top-k list.
        // Everything that is not in the list (block thirds, evicted entries) feeds `dropped`, the largest score
        // left behind; the rescoring pass re-scans the chunk exhaustively when `dropped` reaches its window.
        const int e = threadIdx.x - 128;                    // 0..127 = accumulator row m = 16 * block row + block column
        const int yy = e >> 4, xx = e & 15;
        const float *acc_row = acc_s + e;
        int acc = 0;
        uint32_t tphase = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int chunk = item % p.nchunk, qt = (item / p.nchunk) % n_qt, b = item / (p.nchunk * n_qt);
            const int qy = (qt / p.qt_x) * TQ_R + yy, qx = (qt % p.qt_x) * TV + xx;
            const int rt_b = chunk * p.rt_per_chunk, rt_e = min(n_rt, rt_b + p.rt_per_chunk);
            const float *rinvb = rinv + (size_t)b * p.NR;
            float cv[CORR_TOPK];
            int ci[CORR_TOPK];
            cand_init(cv, ci);
            float dropped = -INFINITY;
            for (int rt = rt_b; rt < rt_e; ++rt) {
                const int ry0 = (rt / p.rt_x) * TR_R, rx0 = (rt % p.rt_x) * TV;
                // per column: score = V * scale + bias, in search units (corr_internal.cuh); bias = -inf: no such patch,
                // or one holding NaN / Inf (rinv NaN; its operands read as 0, so V is finite), which the rescoring scores
                float2 *rc = rcol + acc * UN;
#pragma unroll
                for (int k = 0; k < UN / 128; ++k) {
                    const int n = e + k * 128;
                    const int uu = n >> 4, vv = n & 15;
                    const int ry = ry0 + uu, rx = rx0 + vv;
                    const float ri = vv < TV && ry < p.rh && rx < p.rw ? rinvb[ry * p.rw + rx] : __int_as_float(0x7fffffff);
                    rc[n] = ri == ri ? make_float2(ri, 0.f) : make_float2(0.f, -INFINITY);
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                mbar_wait(tfull, tphase);
                tphase ^= 1;
                const uint32_t rc_s = smem_u32(rc);
#pragma unroll 1
                for (int cc = 0; cc < UN / 32; ++cc) {      // 32 columns = two Ref block rows
                    uint32_t reg[32];
                    acc_ld32(acc_row, cc * 32, UN, reg);
                    float sv[2 * TV];
                    float m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;      // block best, second, third
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                        for (int v = 0; v < TV; ++v) {
                            const int j = hh * 16 + v;
                            // column taps: lane m+dx, column n+dx hold V(q + (0,dx), r + (0,dx))
                            const float t1 = __shfl_down_sync(0xffffffffu, __uint_as_float(reg[j + 1]), 1);
                            const float t2 = __shfl_down_sync(0xffffffffu, __uint_as_float(reg[j + 2]), 2);
                            float cx, cy;
                            asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(cx), "=f"(cy) : "r"(rc_s + (cc * 32 + j) * 8));
                            const float sc = fmaf((__uint_as_float(reg[j]) + t1) + t2, cx, cy);
                            sv[hh * TV + v] = sc;
                            m3 = fmaxf(m3, fminf(m2, sc));
                            m2 = fmaxf(m2, fminf(m1, sc));
                            m1 = fmaxf(m1, sc);
                        }
                    }
                    // the block's two best are offered to the list (neighbouring Ref patches overlap in 6 of 9 pixels,
                    // so the runner-up next to a good match is the likeliest near-tie); the third best is left behind
                    dropped = fmaxf(dropped, m3);
                    if (m1 > cv[3]) {                        // rare once the list has warmed up
                        int k1 = 0, k2 = 0;
#pragma unroll
                        for (int k = 2 * TV - 1; k >= 0; --k)
                            if (sv[k] == m1) k1 = k;                              // lowest column among equals
#pragma unroll
                        for (int k = 2 * TV - 1; k >= 0; --k)
                            if (sv[k] == m2 && k != k1) k2 = k;
                        const int rb = (ry0 + cc * 2) * p.rw + rx0;
                        cand_push(m1, rb + (k1 / TV) * p.rw + k1 % TV, cv, ci, dropped);
                        cand_push(m2, rb + (k2 / TV) * p.rw + k2 % TV, cv, ci, dropped);
                    } else {
                        dropped = fmaxf(dropped, m2);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(tempty);
                acc ^= 1;
            }
            if (xx < TV && qy < p.gh && qx < p.gw)
                part[((size_t)b * p.nchunk + chunk) * p.NQ + qy * p.gw + qx] = cand_pack(cv, ci, dropped);
        }
    }

}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
bool corr_umma_supported(const CorrGeom &g) {
    return g.patch == PATCH && g.s_in == 1 && g.s_ref == 1 && g.w >= BW && g.h >= A_R && g.wr >= BW &&
           g.hr >= B_R;
}

void corr_umma_tiles(const CorrGeom &g, int &n_qt, int &n_rt) {
    n_qt = ceil_div(g.gh, TQ_R) * ceil_div(g.gw, TV);
    n_rt = ceil_div(g.rh, TR_R) * ceil_div(g.rw, TV);
}

// Ref chunks per query tile: the split that minimises (waves over the SMs) x (tiles per item + a fill / drain
// allowance), so small problems (BASELINE config 3: 15 query tiles) still spread over all SMs.
int corr_umma_pick_nchunk(const CorrGeom &g, int sms) {
    int n_qt, n_rt;
    corr_umma_tiles(g, n_qt, n_rt);
    if (sms <= 0) sms = 132;
    int best_n = 1;
    double best_cost = 1e300;
    for (int n = 1; n <= CORR_MAX_CHUNKS && n <= n_rt; ++n) {
        const int per = ceil_div(n_rt, n);
        const int n_eff = ceil_div(n_rt, per);
        if (n_eff != n) continue;                      // no empty chunks
        const long long items = (long long)g.B * n_qt * n;
        const double waves = (double)((items + sms - 1) / sms);
        // + what the exhaustive re-scan of overflowing (query, chunk) pairs costs per query tile: it grows with the chunk
        // length (fitted on the bench step); shorter chunks also mean more list slots
        const double q_tiles = (double)g.B * n_qt;
        const double cost = waves * (per + 0.35) + q_tiles * 2e-3 * per;
        if (cost < best_cost - 1e-9) { best_cost = cost; best_n = n; }
    }
    return best_n;
}

// chunk -> Ref tile range and tile -> Ref patch rectangle, for the exhaustive fallback of the rescoring pass
void corr_umma_chunk_geom(const CorrGeom &g, int nchunk, CorrChunkGeom &cg) {
    cg.mode = 1;
    cg.rt_x = ceil_div(g.rw, TV);
    cg.n_rt = cg.rt_x * ceil_div(g.rh, TR_R);
    cg.per = ceil_div(cg.n_rt, nchunk);
    cg.tile_rows = TR_R;
    cg.tile_cols = TV;
}

int corr_search_umma_launch(const CorrGeom &g, const CorrWorkspace &ws, cudaStream_t st) {
    CUtensorMap tih, til, trh;
    const int C8 = g.Cp / 8;
    int rc;
    if ((rc = make_psa_tensor_map(&tih, ws.hi_in, g.B, C8, g.h, g.w, BW, A_R))) return rc;
    if ((rc = make_psa_tensor_map(&til, ws.lo_in, g.B, C8, g.h, g.w, BW, A_R))) return rc;
    if ((rc = make_psa_tensor_map(&trh, ws.hi_ref, g.B, C8, g.hr, g.wr, BW, B_R))) return rc;

    UmmaParams p;
    p.B = g.B; p.C8 = C8;
    p.gh = g.gh; p.gw = g.gw; p.rh = g.rh; p.rw = g.rw;
    p.qt_x = ceil_div(g.gw, TV); p.qt_y = ceil_div(g.gh, TQ_R);
    p.rt_x = ceil_div(g.rw, TV); p.rt_y = ceil_div(g.rh, TR_R);
    p.nchunk = ws.nchunk;
    p.rt_per_chunk = ceil_div(p.rt_x * p.rt_y, ws.nchunk);
    p.NQ = g.NQ; p.NR = g.NR;

    // per launch: the attribute belongs to the (device, context) pair, not to the process
    C2M_CUDA(cudaFuncSetAttribute(corr_umma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    const int n_items = g.B * p.qt_x * p.qt_y * p.nchunk;
    const int grid = n_items < sms ? n_items : sms;
    corr_umma_kernel<<<grid, 512, SMEM_BYTES, st>>>(tih, til, trh, ws.rinv, ws.part, p);
    C2M_LAUNCH_CHECK("corr_umma_kernel");
    return C2M_OK;
}

}  // namespace c2m
