// Modulated deformable convolution v2 forward on the sm_90a tensor cores (3x3, stride 1, pad 1,
// dilation 1 — every DCN of C2-Matching), fused with DCN_sep_pre_multi_offset's prologue.
//
// Replaces `_ext.dcn_v2_forward` (mmsr/models/archs/DCNv2/src/cuda/dcn_v2_cuda.cu:42-172: im2col
// into a 236-944 MB `columns` buffer + batched fp32 SGEMM) and the Python prologue
// (DCNv2/dcn_v2.py:233-250).  Sampling arithmetic follows dcn_v2_im2col_cuda.cu:25-54,125-195
// operation for operation; the contraction is a split-fp16 (hi*hi + hi*lo + lo*hi) wgmma GEMM
// with fp32 accumulation, i.e. fp32-grade.
//
// Structure = conv3x3_umma.cu with the TMA activation producer replaced by GATHER warps:
//   K is ordered (deformable group g, tap, channel-in-group); a stage = (128-pixel tile, 4 K octets).
//   16 gather warps build the column tile [4 octets][128 px][8] directly in the wgmma K-major
//   no-swizzle layout (hi and lo halves).  A gather thread owns (pixel, run of L K-octets that share one
//   (g, tap) pair), L = min(C/dg/8, 4): the sampling point — raw conv_offset_mask output + pre-offset, sigmoid
//   mask, the 4 corner offsets and mask-folded bilinear weights — is computed ONCE per (pixel, g, tap) and reused
//   for the run's octets; for L > 1 the 4 thread groups work on L consecutive stages concurrently.  Per octet:
//   16 B (hi) + 16 B (lo) per corner, adjacent in the hi/lo-interleaved PSA input (L2 evict-last: the input map is
//   re-read by all nine taps and must stay resident, while offsets bypass L1 and outputs use streaming stores),
//   blended (hi halves in fp32, lo halves in packed fp16), split and stored with one 16 B st.shared per half;
//   fence.proxy.async + mbarrier hand the stage to the MMA warpgroup.
//   Pre-offsets: per tile the index-map cells it can touch ((16/s + 2) x (8/s + 2)) are decoded once into a
//   shared-memory flow table, so the per-(pixel, tap) pre-offset is one ld.shared instead of an 8-byte global
//   load, two integer divisions and a modulo per (pixel, g, tap).
//   Weights stream as 8 KB chunks (bulk copy ring).  A CTA computes one 64-wide slice of the output channels
//   (the fp32 accumulator of a 128 x 64 tile is what one warpgroup holds in registers next to the gather warps);
//   wider layers run their S slices on the S CTAs of a thread-block cluster, which gather each stage once between
//   them and hand it on through distributed shared memory.  The epilogue (bias, LeakyReLU, PSA and / or fp32 store)
//   is shared with the plain convolution.
// The im2col matrix never exists outside shared memory.
#include "umma_conv_common.cuh"

namespace c2m {

namespace {
constexpr int T_R = 16, T_C = 8;
constexpr int KOCT = 4;
constexpr int A_OCT_B = 128 * 16;          // 2048 B: one octet of all 128 pixels (LBO of A)
constexpr int A_HALF = KOCT * A_OCT_B;     // 8192 B
constexpr int A_STAGE = 2 * A_HALF;        // 16384 B
constexpr int MAX_NSTAGE = 8;
constexpr int MAX_NBST = 4;
constexpr int NGATHER_WARPS = 16;
constexpr int NTHREADS = 256 + 32 * NGATHER_WARPS;

struct DcnTc {
    const __half *x_il;        // input, packed-split and hi/lo-interleaved [B][C/8][H][W][hi 8 | lo 8] (value = hi + lo)
    int C8;
    const float *om;           // [B, 3*dg*9, H, W], or octet-planar [B][om_c8][H][W][8] when om_c8 > 0
    int om_c8;
    const float *mask;         // non-null: FINAL modulation mask [B, dg*9, H, W] (no sigmoid) and `om` holds only the
                               // FINAL offsets [B, 2*dg*9, H, W] — the `_ext.dcn_v2_forward` contract
    const unsigned *x_amax;    // [B] bits of the largest finite |x| of each image, or null: x_il holds x * 2^operand_exp
    const unsigned *mask_amax; // [B] the same for the final mask, or null: the gather weights carry mask * 2^mask_exp
    const float *pre;          // [B, 9, H, W, 2] or null
    const long long *idx;      // [B, gh, gw] or null
    int gh, gw, ref_gw, pre_scale;
    int z_end;                 // elements of x_il before its zero tail (B * C * H * W)
    int C, dg, cpg, opp;       // opp = octets per (g, tap) pair = cpg / 8
    int n_ko;                  // real K octets = C/8 * 9
    int L, lshift;             // K octets per gather thread and stage (1, 2 or 4), log2
    int opp_shift;             // log2(opp) when opp is a power of two, else -1 (then L == 1)
    int nstage, nbst;          // ring depths (activation stages, weight chunks); powers of two
    int nstage_shift;          // log2(nstage)
    int slice;                 // 64-wide output-channel slice this launch computes (0 under a cluster launch)
    int sc_shift;              // log2(pre_scale) when the flow table is used (idx given, scale in {1,2,4,8}), else -1
    int tab_h, tab_w;          // flow-table cells per tile: 16/s + 2, 8/s + 2
    float inv_ref_gw, inv_scale;   // reciprocals for the exact float-assisted integer divisions
};
}  // namespace

// exact n / d for 0 <= n < 2^23 with a precomputed float reciprocal (one multiply + fix-up instead
// of the ~25-instruction integer division sequence; the gather loop is issue-bound)
__device__ __forceinline__ int fast_div(int n, int d, float inv_d) {
    int q = (int)((float)n * inv_d);
    const int r = n - q * d;
    q += (r >= d) - (r < 0);
    return q;
}

// ---- cache-policy helpers: the gathered input map is re-read by all nine taps (keep it in L2), the offset /
// mask stream and the outputs are touched once (do not let them evict it)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint4 ldg_keep_v4(const void *ptr, uint64_t pol) {
    uint4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.b32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(ptr), "l"(pol));
    return v;
}
// one (pixel, octet) of the interleaved operand: 32 B = one sector, two 128-bit loads
__device__ __forceinline__ void ldg_keep_v8(const void *ptr, uint64_t pol, uint4 &h, uint4 &l) {
    h = ldg_keep_v4(ptr, pol);
    l = ldg_keep_v4(static_cast<const uint8_t *>(ptr) + 16, pol);
}
__device__ __forceinline__ float2 ldg_stream_f2(const float *ptr, uint64_t pol) {
    float2 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(ptr), "l"(pol));
    return v;
}
__device__ __forceinline__ float ldg_stream_f1(const float *ptr, uint64_t pol) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(ptr), "l"(pol));
    return v;
}

// ---- thread-block cluster helpers (CL = true kernels)
__device__ __forceinline__ uint32_t cluster_reg(int which) {
    uint32_t v;
    if (which == 0) asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(v));
    else if (which == 1) asm("mov.u32 %0, %%cluster_nctarank;" : "=r"(v));
    else if (which == 2) asm("mov.u32 %0, %%clusterid.x;" : "=r"(v));
    else asm("mov.u32 %0, %%nclusterid.x;" : "=r"(v));
    return v;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// shared::cluster address of the same shared-memory object in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t peer_addr(const void *p, int rank) {
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(p)), "r"(rank));
    return a;
}
__device__ __forceinline__ void mbar_arrive_peer(uint32_t bar) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_peer(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.release.cluster.shared::cluster.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}

// CL = false: one launch per 64-wide output-channel slice (d.slice).  CL = true: a cluster of S = nslice CTAs works on
// the same tile sequence, CTA rank r computes slice r, and each gathered stage is built by one CTA and copied into the
// other S - 1 (see the gather-distributor comment below).
template <int N, bool CL>
__global__ void __launch_bounds__(NTHREADS, 1)
dcn_wgmma_kernel(const ConvPtrs q, const ConvParams p, const DcnTc d) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr uint32_t w_half = (uint32_t)KOCT * N * 16;
    constexpr uint32_t w_chunk = 2 * w_half;
    uint8_t *sW = smem;                                   // [nbst][hi | lo]
    uint8_t *sA = smem + d.nbst * w_chunk;                // N multiple of 16 -> multiple of 128
    float *acc_s = reinterpret_cast<float *>(sA + d.nstage * A_STAGE);             // [N][ACC_PITCH]
    uint64_t *bars = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(acc_s) + acc_stage_bytes(N));
    uint64_t *full = bars, *empty = full + MAX_NSTAGE, *bfull = empty + MAX_NSTAGE, *bempty = bfull + MAX_NBST;
    float *sbias = reinterpret_cast<float *>(bempty + MAX_NBST);                  // [N <= 64], 16 B aligned
    int4 *tile_info = reinterpret_cast<int4 *>(sbias + 64);                       // [2] (b, y0, x0, image pixel base)
    float2 *flow_tab = reinterpret_cast<float2 *>(tile_info + 2);                 // [2][tab_h * tab_w]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_img = p.tiles_x * p.tiles_y;
    // Work = flat list of (image, pixel tile), one tile per item (its accumulator lives in the MMA warpgroup's
    // registers); item i runs on CTA i % grid, so at any moment the CTAs work on ~grid CONSECUTIVE tiles and the
    // gathered input map of ONE image is what has to stay in L2, not the whole batch.
    const int n_items = p.B * tiles_img;
    const int nstage_mask = d.nstage - 1;                // ring depths are powers of two (CL: a multiple of S)
    // Clusters: cluster k takes items k, k + nclusters, ... (all its CTAs the same ones), and ring slot i's stages are
    // gathered by CTA i % S, which S | nstage keeps fixed for the whole kernel.
    int rank = 0, S = 1;
    if constexpr (CL) { rank = (int)cluster_reg(0); S = (int)cluster_reg(1); }
    const auto item0 = [&] { return CL ? (int)cluster_reg(2) : (int)blockIdx.x; };
    const auto istep = [&] { return CL ? (int)cluster_reg(3) : (int)gridDim.x; };
    const auto slice = [&] { return CL ? rank : d.slice; };

    if (warp == 1 && lane == 0) {
        for (int i = 0; i < d.nstage; ++i) {
            if (!CL || i % S == rank) {
                mbar_init(&full[i], NGATHER_WARPS >> d.lshift);
                // CL: + 1 elected arrive per MMA warp of each peer, + the distributor once its copies have been read
                mbar_init(&empty[i], CL ? 128 + 4 * (S - 1) + 1 : 128);
            } else {
                mbar_init(&full[i], 1);              // the owner's remote arrive.expect_tx, completed by its bulk copy
                mbar_init(&empty[i], 128);           // arrived on locally, never waited on: the owner's empty[i] gates
            }
        }
        for (int i = 0; i < d.nbst; ++i) { mbar_init(&bfull[i], 1); mbar_init(&bempty[i], 128); }
        fence_mbar_init();
    }
    if constexpr (CL) cluster_sync();       // peers' barriers are initialised before any remote arrive or copy
    else __syncthreads();
    const int sw = *reinterpret_cast<const int *>(q.wblob);

    // Register budget per warpgroup.  The CTA's pool is what it was launched with (80 x 768 = 61440):
    // the control warpgroup gives 56 x 128 back and the MMA / epilogue warpgroup takes them,
    // 24 + 136 + 4 x 80 = 480 = 6 x 80.  Requests beyond the pool would block forever.
    if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (warp == 0) {
        // ================================ weight producer ===================================
        if (lane == 0) {
            int bst = 0, bphase = 0;
            for (int item = item0(); item < n_items; item += istep()) {
                for (int kc = 0; kc < p.nkc; ++kc) {
                    mbar_wait(&bempty[bst], bphase ^ 1);
                    mbar_arrive_expect_tx(&bfull[bst], w_chunk);
                    const uint8_t *src = q.wblob + W_HDR + ((size_t)slice() * p.nkc + kc) * w_chunk;
                    asm volatile(
                        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                        ::"r"(smem_u32(sW + bst * w_chunk)), "l"(src), "r"(w_chunk), "r"(smem_u32(&bfull[bst]))
                        : "memory");
                    if (++bst == d.nbst) { bst = 0; bphase ^= 1; }
                }
            }
        }
    } else if (CL && warp == 1) {
        // ================================ gather distributor (CL) ===========================
        // For each stage this CTA gathered: once its gather warps have completed full[rs], arm every peer's full[rs]
        // for A_STAGE bytes and bulk-copy the slot into the same slot of that peer.  The local empty[rs] gets this
        // thread's arrive only when the copies have finished reading the slot; the peers' MMA warps arrive on it
        // when they have consumed their copy, so the gather warps overwrite the slot only when no CTA still needs it.
        if (lane == 0) {
            int ring = 0;
            for (int item = item0(); item < n_items; item += istep(), ring += p.nkc) {
                for (int kc = (rank - ring % S + S) % S; kc < p.nkc; kc += S) {
                    const int stage_idx = ring + kc;
                    const int rs = stage_idx % d.nstage;
                    mbar_wait(&full[rs], (uint32_t)(stage_idx / d.nstage) & 1u);
                    const uint32_t src = smem_u32(sA + rs * A_STAGE);
                    for (int j = 1; j < S; ++j) {
                        const int peer = (rank + j) % S;
                        const uint32_t pbar = peer_addr(&full[rs], peer);
                        mbar_arrive_expect_tx_peer(pbar, A_STAGE);
                        asm volatile(
                            "cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                            ::"r"(peer_addr(sA + rs * A_STAGE, peer)), "r"(src), "r"(A_STAGE), "r"(pbar)
                            : "memory");
                    }
                    asm volatile("cp.async.bulk.commit_group;\n\tcp.async.bulk.wait_group.read 0;" ::: "memory");
                    mbar_arrive(&empty[rs]);
                }
            }
        }
    }
    } else if (warp < 8) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 136;");
        // ================================ MMA + epilogue ====================================
        // one warpgroup: the wgmmas of both 64-row halves of the tile (A rows 64.. start 8 core-matrix groups in),
        // then the accumulator goes through shared memory to the epilogue, one pixel per thread
        const int e = threadIdx.x - 128;
        const float res_scale = 1.f;
        const float so = ldexpf(1.f, p.sa_out);
        const bool fast = epilogue_fast_ok(q, p) && p.sa_out == 0;     // (this kernel does not pre-scale bias / factors)
        const int o_base = slice() * N;
        for (int i = e; i < N; i += 128) sbias[i] = (q.bias && o_base + i < p.Cout) ? q.bias[o_base + i] : 0.f;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        int stage = 0, phase = 0, bst = 0, bphase = 0;
        for (int item = item0(); item < n_items; item += istep()) {
            const int b = item / tiles_img, tt = item - b * tiles_img;
            const int y = (tt / p.tiles_x) * T_R + e / T_C, x = (tt % p.tiles_x) * T_C + e % T_C;
            const bool ok = y < p.H && x < p.W;
            const float out_scale = ldexpf(1.f, -(operand_exp(d.x_amax, b) + mask_exp(d.mask_amax, b) + sw));
            float acc0[N / 2], acc1[N / 2];                 // rows [0, 64) and [64, 128)
            for (int kc = 0; kc < p.nkc; ++kc) {
                mbar_wait(&bfull[bst], bphase);
                mbar_wait(&full[stage], phase);
                const uint32_t w_hi = smem_u32(sW + bst * w_chunk), w_lo = w_hi + w_half;
                const uint32_t a_hi = smem_u32(sA + stage * A_STAGE), a_lo = a_hi + A_HALF;
                wgmma_fence();
                wgmma_split_chunk128<N, KOCT>(acc0, acc1, a_hi, a_lo, A_OCT_B, w_hi, w_lo, kc);
                wgmma_commit();
                wgmma_wait_all();
                mbar_arrive(&empty[stage]);
                // CL: a stage another CTA gathered is released on that CTA's empty barrier, once per warp (the
                // warp's wgmma reads of it are complete after its wait above)
                if (CL && lane == 0 && stage % S != rank) mbar_arrive_peer(peer_addr(&empty[stage], stage % S));
                mbar_arrive(&bempty[bst]);
                if (++stage == d.nstage) { stage = 0; phase ^= 1; }
                if (++bst == d.nbst) { bst = 0; bphase ^= 1; }
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");          // previous tile's epilogue is done
            acc_store(acc_s, 0, acc0);
            acc_store(acc_s, 64, acc1);
            asm volatile("bar.sync 1, 128;" ::: "memory");
            for (int c0 = 0; c0 < N; c0 += 32) {
                if (fast && c0 + 32 <= N && o_base + c0 + 32 <= p.Cout)
                    epilogue_fast_dispatch(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, nullptr);
                else
                    epilogue_store_block(q, p, acc_s + e, c0, b, y, x, ok, o_base, sbias, out_scale, res_scale, so);
            }
        }
    } else {
        // ================================ gather producers ==================================
        // 4 thread groups of 128 (thread = pixel m of the tile).  With L K-octets per thread a stage has NS = 4 / L
        // thread slots, so the 4 groups split into NG = L stage groups that work on consecutive stages concurrently:
        // group grp -> (stage residue sg = grp / NS, slot = grp % NS); slot covers octets [slot*L, slot*L + L).
        // All index arithmetic is 32-bit (the host checks the map sizes); everything that depends only on the
        // K chunk (group, tap, operand plane offsets) is recomputed when kc changes, not per pixel.
        const int g_tid = threadIdx.x - 256;
        const int m = g_tid & 127;
        const int grp = g_tid >> 7;
        const int L = d.L, NG = L, NS = KOCT >> d.lshift;
        const int sg = grp / NS, slot = grp - sg * NS;
        const int P = p.H * p.W, W8 = p.W * 8;
        const int mrow = m / T_C, mcol = m % T_C;
        const uint64_t pol_keep = l2_policy_evict_last();
        const uint64_t pol_stream = l2_policy_evict_normal();
        const int x_img = d.C8 * P * 8;                       // elements per image of one operand half (< 2^31, host-checked)
        const int om_img = (d.om_c8 > 0 ? d.om_c8 * 8 : (d.mask ? 2 : 3) * d.dg * 9) * P;
        const int om_mask_base = 2 * d.dg * 9;
        const int tab_n = d.tab_h * d.tab_w;
        // cell of this thread's pixel inside a tile's flow table, before the tap shift (+2 halo cells)
        const int cell0 = d.sc_shift >= 0 ? ((mrow >> d.sc_shift) + 2) * d.tab_w + (mcol >> d.sc_shift) + 2 : 0;
        const float Hf = (float)p.H, Wf = (float)p.W;
        struct Meta { float off_h, off_w, mr; };
        int ring = 0;                                       // stages issued by this CTA so far (all groups agree)
        int gi = 0;                                         // item counter (double buffer of tile info and table)
        for (int item = item0(); item < n_items; item += istep(), ++gi) {
            int4 *tinfo = tile_info + (gi & 1);
            float2 *tab = flow_tab + (gi & 1) * tab_n;

            // ---- per item: the tile origin and the decoded flow of every index-map cell the tile can touch
            const int tb = item / tiles_img, tt = item - tb * tiles_img;
            const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
            if (g_tid == 0) *tinfo = make_int4(tb, ty * T_R, tx * T_C, 0);
            if (d.sc_shift >= 0) {
                for (int c = g_tid; c < tab_n; c += 32 * NGATHER_WARPS) {
                    const int cy = c / d.tab_w, cx = c - cy * d.tab_w;
                    const int acy = ((ty * T_R) >> d.sc_shift) - 2 + cy, acx = ((tx * T_C) >> d.sc_shift) - 2 + cx;
                    float2 fl = make_float2(0.f, 0.f);
                    if (acy >= 0 && acx >= 0 && acy < d.gh && acx < d.gw) {
                        const int v = (int)d.idx[((long long)tb * d.gh + acy) * d.gw + acx];
                        const int vy = fast_div(v, d.ref_gw, d.inv_ref_gw), vx = v - vy * d.ref_gw;
                        fl = make_float2((float)((vx - acx) << d.sc_shift), (float)((vy - acy) << d.sc_shift));   // (x, y)
                    }
                    tab[c] = fl;
                }
            }
            asm volatile("bar.sync 2, 512;" ::: "memory");

            // ---- constants of K chunk kc for this thread's octet run
            int c_kc = -1, c_ki = 0, c_kj = 0, c_tap = 0, c_tapcell = 0, c_off = 0, c_moff = 0, c_xoff = 0;
            bool c_valid = false;
            float c_fy = 0.f, c_fx = 0.f;
            auto set_kc = [&](int kc) {
                c_kc = kc;
                const int ko = kc * KOCT + slot * L;
                c_valid = ko < d.n_ko;
                const int pair = d.opp_shift >= 0 ? (ko >> d.opp_shift) : ko / d.opp;
                const int g = pair / 9;
                c_tap = pair - g * 9;
                c_ki = c_tap / 3;
                c_kj = c_tap - c_ki * 3;
                c_fy = (float)(c_ki - 1);
                c_fx = (float)(c_kj - 1);
                c_tapcell = c_ki * d.tab_w + c_kj;
                if (d.om_c8 > 0) {     // octet-planar: channel c of pixel pp lives at ((c >> 3) * P + pp) * 8 + (c & 7)
                    const int c0 = 2 * pair, cm = om_mask_base + pair;
                    c_off = (c0 >> 3) * P * 8 + (c0 & 7);
                    c_moff = (cm >> 3) * P * 8 + (cm & 7);
                } else {
                    c_off = 2 * pair * P;
                    c_moff = (d.mask ? pair : om_mask_base + pair) * P;
                }
                // first channel octet of this run: group g, octets [ko - pair * opp, +L) of the group
                c_xoff = (g * d.opp + (ko - (d.opp_shift >= 0 ? (pair << d.opp_shift) : pair * d.opp))) * P * 8;
            };

            // ---- metadata of K chunk kc: raw offsets (+ pre-offset) and mask logit of this thread's pixel
            auto fetch = [&](int kc, bool in_range, Meta &mt, int &y_out, int &x_out, int &b_out, bool &live) {
                mt.off_h = mt.off_w = mt.mr = 0.f;
                y_out = x_out = b_out = 0;
                live = false;
                if (!in_range) return;
                if (kc != c_kc) set_kc(kc);
                const int4 ti = *tinfo;
                const int b = ti.x, y = ti.y + mrow, xx = ti.z + mcol;
                live = c_valid && y < p.H && xx < p.W;
                y_out = y; x_out = xx; b_out = b;
                if (!live) return;
                const int pp = y * p.W + xx;
                const float *omb = d.om + (size_t)b * om_img;
                if (d.om_c8 > 0) {     // the (y, x) offset pair shares an octet: one 8-byte load
                    const float2 of = ldg_stream_f2(omb + c_off + pp * 8, pol_stream);
                    mt.off_h = of.x;
                    mt.off_w = of.y;
                    mt.mr = ldg_stream_f1(omb + c_moff + pp * 8, pol_stream);
                } else {
                    mt.off_h = ldg_stream_f1(omb + c_off + pp, pol_stream);
                    mt.off_w = ldg_stream_f1(omb + c_off + P + pp, pol_stream);
                    mt.mr = d.mask ? ldg_stream_f1(d.mask + (size_t)b * (d.dg * 9 * P) + c_moff + pp, pol_stream)
                                   : ldg_stream_f1(omb + c_moff + pp, pol_stream);
                }
                if (d.pre) {
                    const float2 pq = *reinterpret_cast<const float2 *>(d.pre + ((size_t)(b * 9 + c_tap) * P + pp) * 2);
                    mt.off_w += pq.x;
                    mt.off_h += pq.y;
                } else if (d.sc_shift >= 0) {
                    const float2 fl = tab[cell0 - c_tapcell];
                    mt.off_w += fl.x;
                    mt.off_h += fl.y;
                } else if (d.idx) {                       // scales the table does not cover: decode in place
                    const int sc = d.pre_scale;
                    const int ys = y - sc * c_ki, xs = xx - sc * c_kj;
                    if (ys >= 0 && xs >= 0) {
                        const int yy = fast_div(ys, sc, d.inv_scale), xg = fast_div(xs, sc, d.inv_scale);
                        if (yy < d.gh && xg < d.gw) {
                            const int v = (int)d.idx[((long long)b * d.gh + yy) * d.gw + xg];
                            const int vy = fast_div(v, d.ref_gw, d.inv_ref_gw), vx = v - vy * d.ref_gw;
                            mt.off_w += (float)(sc * (vx - xg));
                            mt.off_h += (float)(sc * (vy - yy));
                        }
                    }
                }
            };

            // my K chunks of this item: sg, sg + NG, ...  CL: the chunks whose ring slot this CTA owns, the j-th of
            // them for j = sg, sg + NG, ...
            const int kfirst = CL ? (rank - ring % S + S) % S + sg * S : sg;
            const int kstep = CL ? NG * S : NG;
            Meta mt, nx;
            int y, ny, xx, nxx, b, nb;
            bool lv, nlv;
            fetch(kfirst, kfirst < p.nkc, mt, y, xx, b, lv);
            for (int kc = kfirst; kc < p.nkc; kc += kstep) {
                // ---- sampling point of the unit's (pixel, g, tap): dcn_v2_im2col_cuda.cu:25-54,172-190
                const int xoff = lv ? c_xoff : 0;           // belongs to kc (set_kc(kc) ran in this unit's fetch)
                // A corner the sample does not read (outside the image, or the sample outside the window) points at
                // x_il's zero tail: octet u of the run then reads zeros at z_end + u * P * 8, so it contributes exactly
                // 0 whatever the image holds, at no cost per corner.  Offsets reach z_end < 2^31 (host-checked), so
                // their doubling below is unsigned.
                const int zo = d.z_end - (b * x_img + xoff);
                int o0 = zo, o1 = zo, o2 = zo, o3 = zo;
                float w0 = 0.f, w1 = 0.f, w2 = 0.f, w3 = 0.f;
                if (lv) {
                    const float h_im = ((float)y + c_fy) + mt.off_h;
                    const float w_im = ((float)xx + c_fx) + mt.off_w;
                    if (h_im > -1.f && w_im > -1.f && h_im < Hf && w_im < Wf) {
                        const float hf = floorf(h_im), wf = floorf(w_im);
                        const int h_low = (int)hf, w_low = (int)wf;
                        const float lh = h_im - hf, lw = w_im - wf;
                        const float hh = 1.f - lh, hw = 1.f - lw;
                        const bool tv = h_low >= 0, bv = h_low + 1 <= p.H - 1, lvv = w_low >= 0, rv = w_low + 1 <= p.W - 1;
                        // sigmoid to ~2 ulp: the TC path is fp32-grade, not bit-exact; the mask is folded into the weights
                        const float mk = d.mask ? mt.mr * __int_as_float((127 + mask_exp(d.mask_amax, b)) << 23)
                                                : __fdividef(1.f, 1.f + __expf(-mt.mr));
                        const int r0 = h_low * W8 + w_low * 8;
                        const float mh = hh * mk, ml = lh * mk;
                        if (tv && lvv) { o0 = r0; w0 = mh * hw; }
                        if (tv && rv) { o1 = r0 + 8; w1 = mh * lw; }
                        if (bv && lvv) { o2 = r0 + W8; w2 = ml * hw; }
                        if (bv && rv) { o3 = r0 + W8 + 8; w3 = ml * lw; }
                    }
                }
                const __half2 wh0 = __float2half2_rn(w0), wh1 = __float2half2_rn(w1), wh2 = __float2half2_rn(w2),
                              wh3 = __float2half2_rn(w3);
                const int stage_idx = ring + kc;
                const int rs = CL ? stage_idx % d.nstage : stage_idx & nstage_mask;
                const uint32_t rphase = (uint32_t)(CL ? stage_idx / d.nstage : stage_idx >> d.nstage_shift) & 1u;
                uint8_t *sdst = sA + rs * A_STAGE + (slot * L) * A_OCT_B + m * 16;
                // next unit's metadata goes out before this unit's corner fetches come back
                fetch(kc + kstep, kc + kstep < p.nkc, nx, ny, nxx, nb, nlv);
#pragma unroll 1
                for (int u = 0; u < L; ++u) {
                    // octet-planar operand: the 32 lanes of a warp (4 rows x 8 pixels) read 16 B each from runs of
                    // adjacent pixels (8 lines per request instead of 32 with a channels-last fp32 input)
                    const int po = u * P * 8;
                    uint4 ch0, ch1, ch2, ch3, cl0, cl1, cl2, cl3;
                    // element offsets double in the interleaved operand
                    const __half *xi = d.x_il + 2 * ((size_t)b * x_img + xoff + po);
                    ldg_keep_v8(xi + 2u * (unsigned)o0, pol_keep, ch0, cl0);
                    ldg_keep_v8(xi + 2u * (unsigned)o1, pol_keep, ch1, cl1);
                    ldg_keep_v8(xi + 2u * (unsigned)o2, pol_keep, ch2, cl2);
                    ldg_keep_v8(xi + 2u * (unsigned)o3, pol_keep, ch3, cl3);
                    // ---- blend, modulate, split: the hi halves are blended in fp32, the lo halves in packed fp16 —
                    // their rounding lands at 2^-22 of the value
                    const __half2 *hp0 = reinterpret_cast<const __half2 *>(&ch0), *hp1 = reinterpret_cast<const __half2 *>(&ch1);
                    const __half2 *hp2 = reinterpret_cast<const __half2 *>(&ch2), *hp3 = reinterpret_cast<const __half2 *>(&ch3);
                    const __half2 *lp0 = reinterpret_cast<const __half2 *>(&cl0), *lp1 = reinterpret_cast<const __half2 *>(&cl1);
                    const __half2 *lp2 = reinterpret_cast<const __half2 *>(&cl2), *lp3 = reinterpret_cast<const __half2 *>(&cl3);
                    __align__(16) __half2 h4[4];
                    __align__(16) __half2 l4[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        __half2 ls = __hmul2(wh0, lp0[j]);
                        ls = __hfma2(wh1, lp1[j], ls);
                        ls = __hfma2(wh2, lp2[j], ls);
                        ls = __hfma2(wh3, lp3[j], ls);
                        const float2 lf = __half22float2(ls);
                        const float2 a = __half22float2(hp0[j]), bq = __half22float2(hp1[j]);
                        const float2 cq = __half22float2(hp2[j]), dq = __half22float2(hp3[j]);
                        const float vx = fmaf(w0, a.x, fmaf(w1, bq.x, fmaf(w2, cq.x, fmaf(w3, dq.x, lf.x))));
                        const float vy = fmaf(w0, a.y, fmaf(w1, bq.y, fmaf(w2, cq.y, fmaf(w3, dq.y, lf.y))));
                        psa_split2(vx, vy, h4[j], l4[j]);
                    }
                    if (u == 0) mbar_wait(&empty[rs], rphase ^ 1u);
                    *reinterpret_cast<uint4 *>(sdst + u * A_OCT_B) = *reinterpret_cast<const uint4 *>(h4);
                    *reinterpret_cast<uint4 *>(sdst + A_HALF + u * A_OCT_B) = *reinterpret_cast<const uint4 *>(l4);
                }
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) mbar_arrive(&full[rs]);
                mt = nx; lv = nlv; y = ny; xx = nxx; b = nb;
            }
            ring += p.nkc;
        }
    }
    // CL: no CTA exits while a peer can still copy into its shared memory or arrive on its barriers
    if constexpr (CL) cluster_sync();
}

// blob: header | [slice][kc][hi|lo][octet 4][N][8], K ordered (g, tap, channel-in-group)
__global__ void dcn_wpack_kernel(const float *__restrict__ w, int C, int Cout, int dg, int N, int nkc, int nslice,
                                 uint8_t *__restrict__ blob) {
    const int cpg = C / dg, opp = cpg / 8, n_ko = (C / 8) * 9;
    wpack_loop(w, blob, (long long)nslice * nkc * 2 * KOCT * N * 8, [=](long long e, int &half) -> long long {
        const int j = (int)(e & 7);
        long long rest = e >> 3;
        const int ol = (int)(rest % N); rest /= N;
        const int oct = (int)(rest % KOCT); rest /= KOCT;
        half = (int)(rest % 2); rest /= 2;
        const int kc = (int)(rest % nkc);
        const int slice = (int)(rest / nkc);
        const int ko = kc * KOCT + oct, o = slice * N + ol;
        if (ko >= n_ko || o >= Cout) return -1;
        const int pair = ko / opp, oc = ko % opp, g = pair / 9, tap = pair % 9;
        return ((long long)o * C + g * cpg + oc * 8 + j) * 9 + tap;
    });
}

// Largest finite |v| of each image as fp32 bits, for x (blockIdx.z = 0: image b at x + b * nx) and the final mask
// (blockIdx.z = 1: image b at mask + b * nm) in one launch; amax[z * B + b] starts at 0.
__global__ void amax_per_image_kernel(const float *__restrict__ x, long long nx, const float *__restrict__ mask,
                                      long long nm, unsigned *__restrict__ amax) {
    const int b = blockIdx.y, B = gridDim.y;
    const long long n = blockIdx.z ? nm : nx;
    const float *vb = (blockIdx.z ? mask : x) + (size_t)b * n;
    float m = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float a = fabsf(vb[i]);
        if (a < INFINITY) m = fmaxf(m, a);          // NaN and Inf do not set the scale
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax + blockIdx.z * B + b, __float_as_uint(m));
}

// The operand writers below also zero x_il's tail: `tail` pairs of 16-byte halves (hi | lo) after the B*C8*H*W
// pixel octets, which the gather reads for corners it must not read from the image.

// strided fp32 x -> x * 2^operand_exp(image) split into the interleaved operand [B][C8][H][W][hi 8 | lo 8]
// (one thread = one (octet, pixel), pixel fastest: coalesced NCHW reads, one 32 B store)
__global__ void dcn_operand_kernel(const float *__restrict__ x, int C, int C8, int H, int W, long long xs_b,
                                   long long xs_c, long long xs_y, long long xs_x, const unsigned *__restrict__ amax,
                                   long long tail, __half *__restrict__ out) {
    const long long HW = (long long)H * W;
    const long long n = (long long)C8 * HW;
    const int b = blockIdx.y;
    const long long n_here = b == gridDim.y - 1 ? n + tail : n;           // the last image's blocks write the tail
    const float S = ldexpf(1.f, operand_exp(amax, b));
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n_here; e += (long long)gridDim.x * blockDim.x) {
        uint4 *dst = reinterpret_cast<uint4 *>(out + ((size_t)b * n + e) * 16);
        if (e >= n) {
            dst[0] = dst[1] = make_uint4(0, 0, 0, 0);
            continue;
        }
        const int oct = (int)(e / HW);
        const long long pix = e % HW;
        const int y = (int)(pix / W), xx = (int)(pix % W);
        __align__(16) __half h8[16];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = oct * 8 + j;
            psa_split(c < C ? x[b * xs_b + c * xs_c + y * xs_y + xx * xs_x] * S : 0.f, h8[j], h8[8 + j]);
        }
        dst[0] = reinterpret_cast<const uint4 *>(h8)[0];
        dst[1] = reinterpret_cast<const uint4 *>(h8)[1];
    }
}

// PSA hi / lo planes -> the same interleaved operand (and its zero tail): one 32 B sector per corner fetch instead of
// two 16 B halves in separate planes
__global__ void dcn_operand_psa_kernel(const uint4 *__restrict__ hi, const uint4 *__restrict__ lo, long long n,
                                       long long tail, uint4 *__restrict__ out) {
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n + tail; e += (long long)gridDim.x * blockDim.x) {
        const bool body = e < n;
        out[2 * e] = body ? hi[e] : make_uint4(0, 0, 0, 0);
        out[2 * e + 1] = body ? lo[e] : make_uint4(0, 0, 0, 0);
    }
}

static inline int d_pad16(int c) { return (c + 15) / 16 * 16; }
// output channels per launch: a 128 x 64 fp32 accumulator is what the MMA warpgroup keeps in registers
constexpr int D_NMAX = 64;
static inline int d_slice_n(int cout) { return cout <= D_NMAX ? d_pad16(cout) : D_NMAX; }
static inline int d_n_slice(int cout) { return (cout + D_NMAX - 1) / D_NMAX; }
static inline int d_nkc(int C) { return ((C / 8) * 9 + KOCT - 1) / KOCT; }
// K octets per gather thread: the (g, tap) run inside a 4-octet stage when C/dg/8 is a power of two
static inline int d_run(int C, int dg) {
    const int opp = C / dg / 8;
    return (opp & (opp - 1)) ? 1 : (opp >= KOCT ? KOCT : opp);
}

}  // namespace c2m

using namespace c2m;

extern "C" int c2m_dcn_tc_supported(int C, int Cout, int dg) {
    return (C > 0 && Cout > 0 && Cout <= 256 && dg > 0 && C % dg == 0 && (C / dg) % 8 == 0) ? 1 : 0;
}

extern "C" size_t c2m_dcn_tc_packed_weight_bytes(int C, int Cout, int dg) {
    if (!c2m_dcn_tc_supported(C, Cout, dg)) return 0;
    return (size_t)W_HDR + (size_t)d_n_slice(Cout) * d_nkc(C) * 2 * KOCT * d_slice_n(Cout) * 16;
}

extern "C" int c2m_dcn_tc_pack_weights_f32(const float *w, int C, int Cout, int dg, void *packed, c2m_stream_t stream) {
    C2M_CHECK_ARG(w && packed, "dcn_tc_pack_weights: null pointer");
    C2M_CHECK_ARG(c2m_dcn_tc_supported(C, Cout, dg), "dcn_tc_pack_weights: C=%d dg=%d unsupported (C/dg must be a multiple of 8)", C, dg);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (const int rc = wpack_header(w, Cout * C * 9, packed, st)) return rc;
    const int N = d_slice_n(Cout), nkc = d_nkc(C), ns = d_n_slice(Cout);
    const long long total = (long long)ns * nkc * 2 * KOCT * N * 8;
    dcn_wpack_kernel<<<wpack_blocks(total), 256, 0, st>>>(w, C, Cout, dg, N, nkc, ns, reinterpret_cast<uint8_t *>(packed));
    C2M_LAUNCH_CHECK("dcn_wpack_kernel");
    return C2M_OK;
}

// (pixel, octet) pairs of x_il's zero tail: the gather's L-octet runs read it at z_end + u * H * W * 8, u < L
static inline long long d_tail(int C, int dg, int H, int W) { return (long long)(d_run(C, dg) - 1) * H * W + 1; }

extern "C" size_t c2m_dcn_tc_operand_bytes(int B, int C, int H, int W, int dg) {
    if (B <= 0 || H <= 0 || W <= 0 || !c2m_dcn_tc_supported(C, 1, dg)) return 0;
    return ((size_t)B * (C / 8) * H * W + d_tail(C, dg, H, W)) * 32;
}

extern "C" int c2m_dcn_tc_operand_psa(const void *hi, const void *lo, int B, int C, int H, int W, int dg, void *x_il,
                                      c2m_stream_t stream) {
    C2M_CHECK_ARG(hi && lo && x_il && B > 0 && H > 0 && W > 0 && c2m_dcn_tc_supported(C, 1, dg),
                  "dcn_tc_operand_psa: bad argument");
    C2M_CHECK_ARG(((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(x_il) & 31) == 0, "dcn_tc_operand_psa: planes must be 16 B, x_il 32 B aligned");
    const long long n = (long long)B * (C / 8) * H * W, tail = d_tail(C, dg, H, W);
    const long long bx = (n + tail + 255) / 256;
    dcn_operand_psa_kernel<<<(int)(bx > 4096 ? 4096 : bx), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const uint4 *>(hi), reinterpret_cast<const uint4 *>(lo), n, tail, reinterpret_cast<uint4 *>(x_il));
    C2M_LAUNCH_CHECK("dcn_operand_psa_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_tc_operand_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c,
                                      long long xs_y, long long xs_x, int dg, const float *mask, void *x_il,
                                      unsigned *amax, c2m_stream_t stream) {
    C2M_CHECK_ARG(x && x_il && amax && B > 0 && B <= 65535 && H > 0 && W > 0 && c2m_dcn_tc_supported(C, 1, dg),
                  "dcn_tc_operand: bad argument");
    C2M_CHECK_ARG((reinterpret_cast<uintptr_t>(x_il) & 31) == 0, "dcn_tc_operand: x_il must be 32 B aligned");
    // image b must be the C*H*W elements from x + b * C*H*W on (dense NCHW or channels-last): its amax is taken flat.
    // The stride of a dimension of size 1 is never used.
    const long long n = (long long)C * H * W;
    C2M_CHECK_ARG((C == 1 || xs_c > 0) && (H == 1 || xs_y > 0) && (W == 1 || xs_x > 0) && (B == 1 || xs_b == n) &&
                  (C - 1) * xs_c + (H - 1) * xs_y + (W - 1) * xs_x + 1 == n,
                  "dcn_tc_operand: x must be dense NCHW or channels-last");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int nz = mask ? 2 : 1;
    const long long nm = (long long)dg * 9 * H * W;
    C2M_CUDA(cudaMemsetAsync(amax, 0, sizeof(unsigned) * nz * B, st));
    const long long ax = ((n > nm ? n : nm) + 2047) / 2048;
    amax_per_image_kernel<<<dim3(ax > 256 ? 256 : (unsigned)ax, B, nz), 256, 0, st>>>(x, n, mask, nm, amax);
    C2M_LAUNCH_CHECK("amax_per_image_kernel");
    const int C8 = C / 8;
    const long long m = (long long)C8 * H * W, tail = d_tail(C, dg, H, W);
    const long long bx = (m + tail + 255) / 256;
    dcn_operand_kernel<<<dim3((unsigned)(bx > 4096 ? 4096 : bx), B), 256, 0, st>>>(x, C, C8, H, W, B == 1 ? 0 : xs_b,
                                                                                  xs_c, xs_y, xs_x, amax, tail,
                                                                                  reinterpret_cast<__half *>(x_il));
    C2M_LAUNCH_CHECK("dcn_operand_kernel");
    return C2M_OK;
}

extern "C" int c2m_dcn_v2_fused_tc(const c2m_dcn_tc_args *a, c2m_stream_t stream) {
    C2M_CHECK_ARG(a && a->x_il && a->om && a->packed_w, "dcn_v2_fused_tc: null pointer");
    C2M_CHECK_ARG((reinterpret_cast<uintptr_t>(a->x_il) & 31) == 0, "dcn_v2_fused_tc: x_il must be 32 B aligned");
    C2M_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0, "dcn_v2_fused_tc: bad shape");
    C2M_CHECK_ARG(c2m_dcn_tc_supported(a->C, a->Cout, a->dg), "dcn_v2_fused_tc: C=%d dg=%d unsupported", a->C, a->dg);
    C2M_CHECK_ARG(!(a->pre == nullptr && a->idx != nullptr) || (a->gh > 0 && a->gw > 0 && a->ref_gw > 0 && a->pre_scale > 0),
                  "dcn_v2_fused_tc: idx given without a valid grid/scale");
    C2M_CHECK_ARG((a->out_hi == nullptr) == (a->out_lo == nullptr) && (a->out_hi || a->out_f32), "dcn_v2_fused_tc: bad outputs");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    ConvParams p = {};
    p.B = a->B; p.H = a->H; p.W = a->W;
    p.nkc = d_nkc(a->C); p.nkc_a = p.nkc;
    p.Cout = a->Cout; p.N = d_slice_n(a->Cout); p.nslice = d_n_slice(a->Cout);
    p.tiles_x = ceil_div(a->W, T_C); p.tiles_y = ceil_div(a->H, T_R);
    p.act = a->lrelu ? 2 : 0;
    p.sa_in = 0; p.sa_res = 0; p.sa_out = a->sa_out;
    p.ps = 0;
    p.cs = 1;          // streaming output stores: the outputs must not evict the gathered input map from L2
    p.C8out = (a->Cout + 7) / 8; p.Hout = a->H; p.Wout = a->W;
    p.os_b = a->os_b; p.os_c = a->os_c; p.os_y = a->os_y; p.os_x = a->os_x;
    p.f32_mode = a->out_f32 ? f32_store_mode(a->out_f32, nullptr, a->os_b, a->os_c, a->os_y, a->os_x) : 0;
    ConvPtrs q = {};
    q.wblob = reinterpret_cast<const uint8_t *>(a->packed_w);
    q.bias = a->bias;
    q.out_hi = reinterpret_cast<__half *>(a->out_hi); q.out_lo = reinterpret_cast<__half *>(a->out_lo);
    q.out_f32 = a->out_f32;
    DcnTc d;
    d.x_il = reinterpret_cast<const __half *>(a->x_il);
    d.C8 = a->C / 8;
    d.om_c8 = a->om_octets ? (27 * a->dg + 7) / 8 : 0;
    C2M_CHECK_ARG(!a->om_octets || (reinterpret_cast<uintptr_t>(a->om) & 7) == 0, "dcn_v2_fused_tc: om must be 8 B aligned");
    C2M_CHECK_ARG(!a->mask || (!a->om_octets && !a->pre && !a->idx),
                  "dcn_v2_fused_tc: a final mask excludes octet-planar om and pre-offsets");
    d.mask = a->mask;
    d.x_amax = a->x_amax;
    d.mask_amax = a->mask_amax;
    C2M_CHECK_ARG(!a->mask_amax || a->mask, "dcn_v2_fused_tc: mask_amax needs a final mask");
    d.om = a->om; d.pre = a->pre; d.idx = reinterpret_cast<const long long *>(a->idx);
    d.gh = a->gh; d.gw = a->gw; d.ref_gw = a->ref_gw; d.pre_scale = a->pre_scale;
    d.z_end = (int)((long long)a->B * a->C * a->H * a->W);     // < 2^31: checked below, before any launch
    d.C = a->C; d.dg = a->dg; d.cpg = a->C / a->dg; d.opp = d.cpg / 8; d.n_ko = (a->C / 8) * 9;
    d.opp_shift = -1;
    for (int sft = 0; sft < 8; ++sft)
        if (d.opp == (1 << sft)) d.opp_shift = sft;
    d.L = d_run(a->C, a->dg);
    d.lshift = d.L == 4 ? 2 : d.L == 2 ? 1 : 0;
    d.inv_ref_gw = a->ref_gw > 0 ? 1.f / (float)a->ref_gw : 0.f;
    d.inv_scale = a->pre_scale > 0 ? 1.f / (float)a->pre_scale : 1.f;
    // flow table: index-map cells a 16x8 tile (+ the 2-cell tap shift) can touch, when the scale divides the tile
    d.sc_shift = -1;
    d.tab_h = d.tab_w = 0;
    if (!a->pre && a->idx)
        for (int sft = 0; sft < 4; ++sft)
            if (a->pre_scale == (1 << sft)) {
                d.sc_shift = sft;
                d.tab_h = (T_R >> sft) + 2;
                d.tab_w = (T_C >> sft) + 2;
            }
    C2M_CHECK_ARG((long long)a->H * a->W * (27 * a->dg + 7) < (1ll << 31) && (long long)a->H * a->W * a->C < (1ll << 31),
                  "dcn_v2_fused_tc: map too large for 32-bit in-kernel indexing");
    C2M_CHECK_ARG(a->idx == nullptr || (long long)a->gh * a->gw < (1 << 23), "dcn_v2_fused_tc: index map too large");
    C2M_CHECK_ARG((long long)a->B * a->H * a->W * a->C < (1ll << 31), "dcn_v2_fused_tc: batch too large for 32-bit in-kernel indexing");
    // ring depths (powers of two): with L octets per thread, L stage groups fill consecutive stages concurrently.
    // Clusters of S = nslice CTAs: ring slot i belongs to CTA i % S, so the ring is a multiple of S deep (8, or 6 for
    // S = 3), and each CTA gathers into nstage / S of its slots at a time.
    const int S = p.nslice;
    const size_t w_chunk = (size_t)2 * KOCT * p.N * 16;
    d.nstage = S > 1 ? (S == 3 ? 6 : 8) : d.L == 1 ? 4 : 8;
    d.nstage_shift = d.nstage == 4 ? 2 : 3;      // (the cluster kernel indexes the ring with / and %)
    // A stage group's stages are NG * S apart (NG = L).  Its parity wait on empty[] is exact only if the previous
    // stage of the same slot was its own, i.e. NG * S divides nstage: clusters of 3 and 4 use runs of at most 2.
    if (S > 1 && d.L * S > d.nstage) {
        d.L = d.nstage / S;
        d.lshift = d.L == 2 ? 1 : 0;
    }
    const size_t fixed = (size_t)d.nstage * A_STAGE + acc_stage_bytes(p.N) + (2 * MAX_NSTAGE + 2 * MAX_NBST) * 8 + 64 * 4 +
                         2 * 16 + (size_t)2 * d.tab_h * d.tab_w * 8 + 1024 + 128;
    d.nbst = fixed + 4 * w_chunk <= 227 * 1024 ? 4 : 2;
    const size_t smem = fixed + d.nbst * w_chunk;
    C2M_CHECK_ARG(smem <= 227 * 1024, "dcn_v2_fused_tc: %zu bytes of shared memory needed", smem);
    C2M_CUDA(cudaFuncSetAttribute(dcn_wgmma_kernel<16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    C2M_CUDA(cudaFuncSetAttribute(dcn_wgmma_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    C2M_CUDA(cudaFuncSetAttribute(dcn_wgmma_kernel<48, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    C2M_CUDA(cudaFuncSetAttribute(dcn_wgmma_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    C2M_CUDA(cudaFuncSetAttribute(dcn_wgmma_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    const long long n_items = (long long)a->B * p.tiles_x * p.tiles_y;
    C2M_CHECK_ARG(n_items < (1 << 23), "dcn_v2_fused_tc: too many pixel tiles");
    // SURVEY.md §8(d): flops = 2*B*Cout*C*9*Ho*Wo; bytes = 4*B*(C*H*W + 3*dg*9*H*W + Cout*H*W) + weights
    const double px = (double)a->B * a->H * a->W;
    const double flops = 2.0 * a->Cout * a->C * 9.0 * px;
    const double bytes = 4.0 * px * (a->C + 27.0 * a->dg + a->Cout) + 4.0 * a->Cout * (a->C * 9.0 + 1.0);
    d.slice = 0;
    if (S == 1) {
        void *ph = prof_begin(PROF_DCN, flops, bytes, st);
        const int grid = n_items < sms ? (int)n_items : sms;
        switch (p.N) {
        case 16: dcn_wgmma_kernel<16, false><<<grid, NTHREADS, smem, st>>>(q, p, d); break;
        case 32: dcn_wgmma_kernel<32, false><<<grid, NTHREADS, smem, st>>>(q, p, d); break;
        case 48: dcn_wgmma_kernel<48, false><<<grid, NTHREADS, smem, st>>>(q, p, d); break;
        default: dcn_wgmma_kernel<64, false><<<grid, NTHREADS, smem, st>>>(q, p, d); break;
        }
        C2M_LAUNCH_CHECK("dcn_wgmma_kernel");
        prof_end(ph, st);
        return C2M_OK;
    }
    // Cout > 64: the S slices of a tile run at once on the CTAs of one cluster, which gather it once between them
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)S;
    attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(S * (sms / S)));
    cfg.blockDim = dim3(NTHREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int nclusters = 0;
    C2M_CUDA(cudaOccupancyMaxActiveClusters(&nclusters, dcn_wgmma_kernel<64, true>, &cfg));
    C2M_CHECK_ARG(nclusters > 0, "dcn_v2_fused_tc: no cluster of %d CTAs with %zu bytes of shared memory fits", S, smem);
    if (nclusters > n_items) nclusters = (int)n_items;
    cfg.gridDim = dim3((unsigned)(S * nclusters));
    void *ph = prof_begin(PROF_DCN, flops, bytes, st);
    C2M_CUDA(cudaLaunchKernelEx(&cfg, dcn_wgmma_kernel<64, true>, q, p, d));
    C2M_LAUNCH_CHECK("dcn_wgmma_kernel");
    prof_end(ph, st);
    return C2M_OK;
}
