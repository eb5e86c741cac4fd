// Backward of the tensor-core deformable convolution (dcn_umma.cu, the `_ext` contract: final offsets, final mask,
// 3x3 / stride 1 / pad 1 / dilation 1, one conv group) on the sm_90a tensor cores, fp32-grade (split fp16 x 3).
//
// Both kernels work on the forward's 16x8-pixel tiles and its column order K = (deformable group g, tap, channel in
// group).  grad_output enters as PSA at the per-image power-of-two scale 2^sg_b of c2m_conv3x3_operand_f32; x enters as
// the forward's
// interleaved operand x_il (x * 2^sa_b per image) and the final mask as mask * 2^sm_b (c2m_dcn_tc_operand_f32).  Every
// result is divided by its own image's exponents, so an image's gradients do not depend on the other images.
//
// dcn_dgrad_kernel: gcol = W^T gY, M = the tile's 128 pixels, N = a chunk of columns, K = Cout.  gY arrives by TMA as
// the forward's K-major activation layout [octet][128 px][8], the weights as a second packed blob (K = Cout octets,
// N = columns).  The MMA warpgroup hands each finished chunk to one of three epilogue warpgroups through shared
// memory; the chunks of one (g, tap) pair all go to the same warpgroup, so the thread of a pixel owns (pixel, g, tap):
// it recomputes the sampling point with dcn_sample_point / DcnCorners, reads the four corners of the group's channels
// from x_il (one 32 B sector per corner octet), and sums grad_mask and grad_offset in one fixed order (channel octet,
// corner, channel) with the formulas of dcn_col2im_coord_kernel, writing each element once.  The GI variant also scatters
// grad_input with atomics (dcn_col2im_kernel's sum).  gcol never leaves the chip.
//
// dcn_wgrad_kernel: dW = gY col^T, M = Cout (a slice of up to 128), N = one 4-octet column stage, K = pixels.  Gather
// warps build mask * bilinear(x) for a tile in the forward's [octet][px][8] layout, which is an MN-major operand along
// K = pixels; gY is the MN-major operand of the same tile by TMA (as in conv3x3_wgrad.cu).  The accumulator is added
// into the CTA's fp32 workspace slot every WG_FLUSH tiles and whenever the image changes, divided by that image's
// operand scales 2^(sa_b + sm_b + sg_b); wgrad_reduce_kernel sums the slots in one fixed order
// (umma_conv_common.cuh).
#include "dcn_sampling.cuh"
#include "umma_conv_common.cuh"

namespace c2m {

namespace {
constexpr int T_R = 16, T_C = 8;                 // pixel tile (the forward's)
constexpr int OCT_B = 128 * 16;                  // one channel octet of a tile's 128 pixels: 2048 B
constexpr int KOCT = 4;                          // channel octets per K piece (dgrad) / per column stage (wgrad)
constexpr int PIECE_HALF = KOCT * OCT_B;         // 8192 B
constexpr int NTHREADS = 768;
// dgrad
constexpr int DG_NMAX = 64;                      // columns per chunk (a 128 x 64 fp32 accumulator in one warpgroup)
constexpr int DG_NEPI = 3;                       // epilogue warpgroups, one staging buffer each
constexpr int DG_THREADS = 256 + 128 * DG_NEPI;
constexpr int DG_NST = 4;                        // (gY piece, weight piece) ring
constexpr int DG_STAGE = 2 * PIECE_HALF + 2 * KOCT * DG_NMAX * 16;
constexpr size_t DG_SMEM = (size_t)DG_NST * DG_STAGE + (size_t)DG_NEPI * acc_stage_bytes(DG_NMAX) +
                           (2 * DG_NST + 2 * DG_NEPI) * 8 + 1024;
// wgrad
constexpr int WG_NCO = 128;                      // output channels one gather serves
constexpr int WG_NSY = 2, WG_NSG = 4;            // gY ring, column ring
constexpr int WG_COL_STAGE = 2 * PIECE_HALF;     // 4 octets x 128 px, hi | lo
constexpr int WG_FLUSH = 8;                      // tiles per accumulator run (8 K steps x 3 MMAs each)

struct DcnGrad {
    const __half *x_il;
    const unsigned *x_amax, *mask_amax, *gy_amax;
    const float *off, *mask;
    const uint8_t *wblob;
    float *goff, *gmask, *gx, *ws;
    int B, C, H, W, Cout, dg, cpg, opp, C8, C8o;
    int tiles_x, tiles_y;
    int N, nch, cpc, nkp;                  // dgrad: columns per chunk, chunks, chunks per (g, tap) pair, K pieces
    int n_ko;                              // real column octets (C / 8 * 9)
    int nkc, nh, ncs, ksplit;              // wgrad: column stages, m64 halves per slice, slices, K ranges
    long long ntiles;
    c2m_dcn_shape s;                       // geometry for dcn_sample_point
};

// one corner octet of the interleaved operand (hi 8 | lo 8 = one 32 B sector) as 8 fp32 values
__device__ __forceinline__ void ld_octet_f32(const __half *x_il, size_t pix, float (&v)[8]) {
    const uint4 *src = reinterpret_cast<const uint4 *>(x_il) + pix * 2;
    psa_unsplit2(__ldg(src), __ldg(src + 1), v);
}
}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// dgrad.  Warp 0 streams (gY piece, weight piece) stages; warpgroup 1 runs the MMAs of one chunk and stores the
// accumulator into staging buffer e of the chunk's epilogue warpgroup e = (chunk / cpc) % 3; warpgroups 2..4 are the
// epilogues (thread = pixel of the tile).
// ------------------------------------------------------------------------------------------------------------------
template <int N, bool GI>
__global__ void __launch_bounds__(DG_THREADS, 1) dcn_dgrad_kernel(const __grid_constant__ CUtensorMap tg_hi,
                                                                const __grid_constant__ CUtensorMap tg_lo,
                                                                const DcnGrad d) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr uint32_t w_half = (uint32_t)KOCT * N * 16;
    float *stg = reinterpret_cast<float *>(smem + DG_NST * DG_STAGE);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + DG_NST * DG_STAGE + DG_NEPI * acc_stage_bytes(DG_NMAX));
    uint64_t *empty = full + DG_NST, *sfull = empty + DG_NST, *sempty = sfull + DG_NEPI;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_img = d.tiles_x * d.tiles_y;
    const int n_items = (int)d.ntiles;
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tg_hi);
        tma_prefetch_desc(&tg_lo);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < DG_NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 128); }
        for (int i = 0; i < DG_NEPI; ++i) { mbar_init(&sfull[i], 128); mbar_init(&sempty[i], 128); }
        fence_mbar_init();
    }
    __syncthreads();

    // register pool of the launch, 5 x 96 per thread slot: producer 40 + MMA 128 + 3 x 104 epilogue
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            int st = 0, ph = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int b = item / tiles_img, tt = item - b * tiles_img;
                const int y0 = (tt / d.tiles_x) * T_R, x0 = (tt % d.tiles_x) * T_C;
                for (int ch = 0; ch < d.nch; ++ch)
                    for (int kp = 0; kp < d.nkp; ++kp) {
                        mbar_wait(&empty[st], ph ^ 1);
                        uint8_t *s = smem + st * DG_STAGE;
                        mbar_arrive_expect_tx(&full[st], 2 * PIECE_HALF + 2 * w_half);
                        tma_load_4d(s, &tg_hi, &full[st], x0 * 8, y0, kp * KOCT, b);
                        tma_load_4d(s + PIECE_HALF, &tg_lo, &full[st], x0 * 8, y0, kp * KOCT, b);
                        const uint8_t *src = d.wblob + W_HDR + ((size_t)ch * d.nkp + kp) * 2 * w_half;
                        asm volatile(
                            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                            ::"r"(smem_u32(s + 2 * PIECE_HALF)), "l"(src), "r"(2 * w_half), "r"(smem_u32(&full[st]))
                            : "memory");
                        if (++st == DG_NST) { st = 0; ph ^= 1; }
                    }
            }
        }
    } else if (warp < 8) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 128;");
        // ================================ MMA ================================
        int st = 0, ph = 0;
        uint32_t sent = 0;                                  // bit e: parity of the chunks handed to epilogue e
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            for (int ch = 0; ch < d.nch; ++ch) {
                float acc0[N / 2], acc1[N / 2];            // pixel rows [0, 64) and [64, 128)
                for (int kp = 0; kp < d.nkp; ++kp) {
                    mbar_wait(&full[st], ph);
                    const uint32_t a_hi = smem_u32(smem + st * DG_STAGE), a_lo = a_hi + PIECE_HALF;
                    const uint32_t w_hi = a_hi + 2 * PIECE_HALF, w_lo = w_hi + w_half;
                    wgmma_fence();
                    wgmma_split_chunk128<N, KOCT>(acc0, acc1, a_hi, a_lo, OCT_B, w_hi, w_lo, kp);
                    wgmma_commit();
                    wgmma_wait_all();
                    mbar_arrive(&empty[st]);
                    if (++st == DG_NST) { st = 0; ph ^= 1; }
                }
                const int e = (ch / d.cpc) % DG_NEPI;
                mbar_wait(&sempty[e], ((sent >> e) & 1u) ^ 1u);
                float *buf = stg + e * (acc_stage_bytes(DG_NMAX) / 4);
                acc_store(buf, 0, acc0);
                acc_store(buf, 64, acc1);
                mbar_arrive(&sfull[e]);
                sent ^= 1u << e;
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 104;");
        // ================================ epilogues ================================
        const int e = (threadIdx.x - 256) >> 7, m = threadIdx.x & 127;
        const float *buf = stg + e * (acc_stage_bytes(DG_NMAX) / 4) + m;
        const size_t plane = (size_t)d.H * d.W;
        const int sw_blob = *reinterpret_cast<const int *>(d.wblob);
        int got = 0;
        float sh = 0.f, sw = 0.f, sm = 0.f;                 // running sums of the current (pixel, g, tap)
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int b = item / tiles_img, tt = item - b * tiles_img;
            const int y = (tt / d.tiles_x) * T_R + m / T_C, x = (tt % d.tiles_x) * T_C + m % T_C;
            const bool ok = y < d.H && x < d.W;
            const int p = y * d.W + x;
            const int sgw = grad_scale_exp(d.gy_amax + b) + sw_blob;    // gcol = 2^sgw W^T gY of image b
            // unscaled as one ldexpf of the result: 2^-(sgw + sa_b) alone can be below fp32's range
            const int out_exp = -(sgw + operand_exp(d.x_amax, b));
            const float *offb = d.off + (size_t)b * 2 * d.dg * 9 * plane;
            const float *maskb = d.mask + (size_t)b * d.dg * 9 * plane;
            for (int ch = 0; ch < d.nch; ++ch) {
                if ((ch / d.cpc) % DG_NEPI != e) continue;
                mbar_wait(&sfull[e], got & 1);
                ++got;
                if (ok) {
                    // column octets of this chunk (the last chunk may end early: its padding columns are zero)
                    const int k0 = ch * d.N / 8, k1 = min(k0 + d.N / 8, d.n_ko);
                    for (int k = k0; k < k1;) {
                        const int pair = k / d.opp, oc0 = k - pair * d.opp;
                        const int kend = min(k1, (pair + 1) * d.opp);
                        const int g = pair / 9, tap = pair - g * 9;
                        const float mk = maskb[pair * plane + p];
                        float h_im, w_im;
                        const bool in = dcn_sample_point(d.s, d.W, tap, p, offb[2 * pair * plane + p],
                                                         offb[(2 * pair + 1) * plane + p], h_im, w_im);
                        const DcnCorners<float> q(h_im, w_im, d.H, d.W, d.W, 1);
                        const float hh = 1.f - q.lh, hw = 1.f - q.lw;
                        if (oc0 == 0) sh = sw = sm = 0.f;
                        if (in) {
                            for (int oc = oc0; oc < oc0 + (kend - k); ++oc) {
                                const size_t xo = ((size_t)b * d.C8 + g * d.opp + oc) * plane;
                                const float *gcp = buf + (size_t)((k - k0) + (oc - oc0)) * 8 * ACC_PITCH;
                                float gc[8];
#pragma unroll
                                for (int j = 0; j < 8; ++j) gc[j] = gcp[j * ACC_PITCH];
                                // corner by corner: d(sample)/dh and d(sample)/dw of corner c are dh[c] and dw[c]
                                const float dh[4] = {-hw, -q.lw, hw, q.lw}, dw[4] = {-hh, hh, -q.lh, q.lh};
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    if (!q.ok[c]) continue;
                                    float v[8];
                                    ld_octet_f32(d.x_il, xo + q.o[c], v);
#pragma unroll
                                    for (int j = 0; j < 8; ++j) {
                                        const float gv = gc[j] * v[j];
                                        sm += gv * q.w[c];
                                        sh += gv * dh[c];
                                        sw += gv * dw[c];
                                    }
                                    if (GI) {
                                        float *gim = d.gx + ((size_t)b * d.C + (g * d.opp + oc) * 8) * plane + q.o[c];
#pragma unroll
                                        for (int j = 0; j < 8; ++j) atomicAdd(gim + j * plane, ldexpf(gc[j] * mk * q.w[c], -sgw));
                                    }
                                }
                            }
                        }
                        if (kend == (pair + 1) * d.opp) {           // last octet of the pair: write its gradients
                            const size_t j0 = (size_t)(b * d.dg * 9 + pair);
                            d.goff[(2 * j0) * plane + p] = in ? ldexpf(sh * mk, out_exp) : 0.f;
                            d.goff[(2 * j0 + 1) * plane + p] = in ? ldexpf(sw * mk, out_exp) : 0.f;
                            d.gmask[j0 * plane + p] = in ? ldexpf(sm, out_exp) : 0.f;
                        }
                        k = kend;
                    }
                }
                mbar_arrive(&sempty[e]);
            }
        }
    }
}

// blob: header | [chunk][K piece][hi|lo][octet 4][N][8]: column n of chunk ch is K4's K index ch * N + n (zero past
// C * 9, in the last chunk), row (octet, j) of piece kp is output channel (kp * 4 + octet) * 8 + j
__global__ void dcn_dgrad_wpack_kernel(const float *__restrict__ w, int C, int Cout, int dg, int N, int nch, int nkp,
                                       uint8_t *__restrict__ blob) {
    const int cpg = C / dg;
    wpack_loop(w, blob, (long long)nch * nkp * 2 * KOCT * N * 8, [=](long long e, int &half) -> long long {
        const int j = (int)(e & 7);
        long long rest = e >> 3;
        const int n = (int)(rest % N); rest /= N;
        const int oct = (int)(rest % KOCT); rest /= KOCT;
        half = (int)(rest % 2); rest /= 2;
        const int kp = (int)(rest % nkp);
        const int ch = (int)(rest / nkp);
        const int co = (kp * KOCT + oct) * 8 + j, col = ch * N + n;
        const int pair = col / cpg, g = pair / 9, tap = pair % 9, c = g * cpg + col % cpg;
        return co < Cout && col < C * 9 ? ((long long)co * C + c) * 9 + tap : -1;
    });
}

// ------------------------------------------------------------------------------------------------------------------
// wgrad.  CTA = (column stage kc, output-channel slice cs, tile range k), kc fastest.  Warp 0 streams gY tiles by TMA;
// warpgroup 1 runs the MMAs; warpgroups 2..5 gather (thread = pixel m x column octet u of the stage).
// ------------------------------------------------------------------------------------------------------------------
template <int NH>
__global__ void __launch_bounds__(NTHREADS, 1) dcn_wgrad_kernel(const __grid_constant__ CUtensorMap tg_hi,
                                                                const __grid_constant__ CUtensorMap tg_lo,
                                                                const DcnGrad d) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int Y_HALF = NH * 8 * OCT_B;
    uint8_t *sY = smem;                                      // [WG_NSY][hi | lo][NH * 8 octets][128 px][8]
    uint8_t *sG = smem + WG_NSY * 2 * Y_HALF;                // [WG_NSG][hi | lo][4 octets][128 px][8]
    uint64_t *yfull = reinterpret_cast<uint64_t *>(sG + WG_NSG * WG_COL_STAGE), *yempty = yfull + WG_NSY;
    uint64_t *gfull = yempty + WG_NSY, *gempty = gfull + WG_NSG;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kc = blockIdx.x % d.nkc;
    const int cs = (blockIdx.x / d.nkc) % d.ncs;
    const int kr = blockIdx.x / (d.nkc * d.ncs);
    const long long t0 = d.ntiles * kr / d.ksplit, t1 = d.ntiles * (kr + 1) / d.ksplit;
    const int tiles_img = d.tiles_x * d.tiles_y;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tg_hi);
        tma_prefetch_desc(&tg_lo);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < WG_NSY; ++i) { mbar_init(&yfull[i], 1); mbar_init(&yempty[i], 128); }
        for (int i = 0; i < WG_NSG; ++i) { mbar_init(&gfull[i], 16); mbar_init(&gempty[i], 128); }
        fence_mbar_init();
    }
    __syncthreads();

    // register pool of the launch, 6 x 80 per thread slot: producer 40 + MMA 120 + 4 x 80 gather
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            // boxes of 4 octets that hold real channels of this slice
            const int oct0 = cs * NH * 8;
            const int nbox = min(NH * 2, (d.C8o - oct0 + KOCT - 1) / KOCT);
            int st = 0, ph = 0;
            for (long long t = t0; t < t1; ++t) {
                const int b = (int)(t / tiles_img), tt = (int)(t % tiles_img);
                const int y0 = (tt / d.tiles_x) * T_R, x0 = (tt % d.tiles_x) * T_C;
                mbar_wait(&yempty[st], ph ^ 1);
                uint8_t *s = sY + st * 2 * Y_HALF;
                mbar_arrive_expect_tx(&yfull[st], nbox * 2 * PIECE_HALF);
                for (int bx = 0; bx < nbox; ++bx) {
                    tma_load_4d(s + bx * PIECE_HALF, &tg_hi, &yfull[st], x0 * 8, y0, oct0 + bx * KOCT, b);
                    tma_load_4d(s + Y_HALF + bx * PIECE_HALF, &tg_lo, &yfull[st], x0 * 8, y0, oct0 + bx * KOCT, b);
                }
                if (++st == WG_NSY) { st = 0; ph ^= 1; }
            }
        }
    } else if (warp < 8) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 120;");
        // ================================ MMA ================================
        float acc[NH][16];
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
        const int ncol = d.nkc * 32;
        float *blk = d.ws + ((size_t)kr * d.ncs * WG_NCO + cs * WG_NCO) * ncol + kc * 32;
        bool first = true;
        auto flush = [&](int b) {
            wgrad_flush(acc, blk, ncol, 64 * ncol, first,
                        -(operand_exp(d.x_amax, b) + mask_exp(d.mask_amax, b) + grad_scale_exp(d.gy_amax + b)));
            first = false;
        };
        int ys = 0, yph = 0, gs = 0, gph = 0, n = 0, cur_b = -1;
        for (long long t = t0; t < t1; ++t) {
            const int b = (int)(t / tiles_img);
            if (n > 0 && (b != cur_b || n == WG_FLUSH)) { flush(cur_b); n = 0; }
            cur_b = b;
            mbar_wait(&yfull[ys], yph);
            mbar_wait(&gfull[gs], gph);
            const uint32_t yh = smem_u32(sY + ys * 2 * Y_HALF), yl = yh + Y_HALF;
            const uint32_t ch = smem_u32(sG + gs * WG_COL_STAGE), cl = ch + PIECE_HALF;
            // MN-major descriptors: lbo = next 8 pixels along K, sbo = next octet along M / N
            const uint64_t dch = wg_smem_desc(ch, 128, OCT_B), dcl = wg_smem_desc(cl, 128, OCT_B);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 8; ++j) {                    // K step j: pixels [16 j, 16 j + 16)
#pragma unroll
                for (int h = 0; h < NH; ++h) {
                    wgmma_tt_split(acc[h], wg_smem_desc(yh + h * 8 * OCT_B + j * 256, 128, OCT_B),
                                   wg_smem_desc(yl + h * 8 * OCT_B + j * 256, 128, OCT_B), wg_desc_advance(dch, j * 256),
                                   wg_desc_advance(dcl, j * 256));
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            mbar_arrive(&yempty[ys]);
            mbar_arrive(&gempty[gs]);
            if (++ys == WG_NSY) { ys = 0; yph ^= 1; }
            if (++gs == WG_NSG) { gs = 0; gph ^= 1; }
            ++n;
        }
        if (n > 0) flush(cur_b);
    } else {
        // ================================ gather ================================
        const int gt = threadIdx.x - 256, m = gt & 127, u = gt >> 7;
        const int ko = kc * KOCT + u;
        const bool valid = ko < d.n_ko;
        const int pair = valid ? ko / d.opp : 0, oc = ko - pair * d.opp;
        const int g = pair / 9, tap = pair - g * 9;
        const size_t plane = (size_t)d.H * d.W;
        int gs = 0, gph = 0;
        for (long long t = t0; t < t1; ++t) {
            const int b = (int)(t / tiles_img), tt = (int)(t % tiles_img);
            const int y = (tt / d.tiles_x) * T_R + m / T_C, x = (tt % d.tiles_x) * T_C + m % T_C;
            float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (valid && y < d.H && x < d.W) {
                const int p = y * d.W + x;
                const size_t j0 = (size_t)b * d.dg * 9 + pair;
                float h_im, w_im;
                if (dcn_sample_point(d.s, d.W, tap, p, d.off[2 * j0 * plane + p], d.off[(2 * j0 + 1) * plane + p],
                                     h_im, w_im)) {
                    const float mk = d.mask[j0 * plane + p] * __int_as_float((127 + mask_exp(d.mask_amax, b)) << 23);
                    const DcnCorners<float> q(h_im, w_im, d.H, d.W, d.W, 1);
                    const size_t xo = ((size_t)b * d.C8 + g * d.opp + oc) * plane;
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (q.ok[c]) {
                            float cv[8];
                            ld_octet_f32(d.x_il, xo + q.o[c], cv);
                            const float wc = q.w[c] * mk;
#pragma unroll
                            for (int j = 0; j < 8; ++j) v[j] = fmaf(wc, cv[j], v[j]);
                        }
                }
            }
            __align__(16) __half2 h4[4];
            __align__(16) __half2 l4[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) psa_split2(v[2 * j], v[2 * j + 1], h4[j], l4[j]);
            mbar_wait(&gempty[gs], gph ^ 1);
            uint8_t *dst = sG + gs * WG_COL_STAGE + u * OCT_B + m * 16;
            *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<const uint4 *>(h4);
            *reinterpret_cast<uint4 *>(dst + PIECE_HALF) = *reinterpret_cast<const uint4 *>(l4);
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&gfull[gs]);
            if (++gs == WG_NSG) { gs = 0; gph ^= 1; }
        }
    }
}

// ---- host side
// columns per dgrad chunk: whole (g, tap) pairs when a pair has at most 64 columns (the last chunk is then partial
// unless the pair count divides evenly), else the largest wgmma width dividing the pair, so that no chunk holds parts
// of two pairs
static int dg_chunk_n(int cpg) {
    if (cpg <= DG_NMAX) return (DG_NMAX / cpg) * cpg;
    for (int n = DG_NMAX; n > 8; n -= 8)
        if (cpg % n == 0) return n;
    return 8;
}

static int grad_geom(int B, int C, int H, int W, int Cout, int dg, DcnGrad &d) {
    d = DcnGrad{};
    d.B = B; d.C = C; d.H = H; d.W = W; d.Cout = Cout; d.dg = dg;
    d.cpg = C / dg; d.opp = d.cpg / 8; d.C8 = C / 8; d.C8o = (Cout + 7) / 8;
    d.tiles_x = ceil_div(W, T_C); d.tiles_y = ceil_div(H, T_R);
    d.ntiles = (long long)B * d.tiles_x * d.tiles_y;
    d.N = dg_chunk_n(d.cpg);
    d.nch = ceil_div(C * 9, d.N);
    d.cpc = d.cpg > DG_NMAX ? d.cpg / d.N : 1;
    d.nkp = ceil_div(d.C8o, KOCT);
    d.n_ko = d.C8 * 9;
    d.nkc = ceil_div(d.n_ko, KOCT);
    d.nh = Cout <= 64 ? 1 : 2;
    d.ncs = ceil_div(Cout, WG_NCO);
    c2m_dcn_shape &s = d.s;
    s = c2m_dcn_shape{};
    s.B = B; s.C = C; s.H = H; s.W = W; s.Cout = Cout; s.kh = s.kw = 3; s.sh = s.sw = 1; s.ph = s.pw = 1;
    s.dh = s.dw = 1; s.dg = dg;
    return C2M_OK;
}

// shape and operand checks shared by both entry points
static int check_grad_args(const c2m_dcn_tc_grad_args *a, const char *who) {
    C2M_CHECK_ARG(a, "%s: null arguments", who);
    C2M_CHECK_ARG(a->gy_hi && a->gy_lo && a->gy_amax && a->x_il && a->x_amax && a->mask_amax && a->offset && a->mask,
                  "%s: null pointer", who);
    C2M_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0, "%s: bad shape", who);
    C2M_CHECK_ARG(c2m_dcn_tc_supported(a->C, a->Cout, a->dg), "%s: C=%d Cout=%d dg=%d unsupported", who, a->C, a->Cout,
                  a->dg);
    C2M_CHECK_ARG(a->H >= T_R && a->W >= T_C, "%s: map %dx%d smaller than one pixel tile (16x8)", who, a->H, a->W);
    C2M_CHECK_ARG((long long)a->B * a->C * a->H * a->W < (1ll << 31) && (long long)a->B * 27 * a->dg * a->H * a->W < (1ll << 31),
                  "%s: tensors too large for 32-bit in-kernel indexing", who);
    C2M_CHECK_ARG((reinterpret_cast<uintptr_t>(a->x_il) & 31) == 0, "%s: x_il must be 32 B aligned", who);
    return C2M_OK;
}

}  // namespace c2m

using namespace c2m;

extern "C" size_t c2m_dcn_tc_dgrad_packed_weight_bytes(int C, int Cout, int dg) {
    if (!c2m_dcn_tc_supported(C, Cout, dg)) return 0;
    const int cpg = C / dg, N = dg_chunk_n(cpg);
    return (size_t)W_HDR + (size_t)ceil_div(C * 9, N) * ceil_div((Cout + 7) / 8, KOCT) * 2 * KOCT * N * 16;
}

extern "C" int c2m_dcn_tc_pack_dgrad_weights_f32(const float *w, int C, int Cout, int dg, void *packed,
                                                 c2m_stream_t stream) {
    C2M_CHECK_ARG(w && packed, "dcn_tc_pack_dgrad_weights: null pointer");
    C2M_CHECK_ARG(c2m_dcn_tc_supported(C, Cout, dg), "dcn_tc_pack_dgrad_weights: C=%d Cout=%d dg=%d unsupported", C,
                  Cout, dg);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (const int rc = wpack_header(w, Cout * C * 9, packed, st)) return rc;
    const int N = dg_chunk_n(C / dg), nch = ceil_div(C * 9, N), nkp = ceil_div((Cout + 7) / 8, KOCT);
    const long long total = (long long)nch * nkp * 2 * KOCT * N * 8;
    dcn_dgrad_wpack_kernel<<<wpack_blocks(total), 256, 0, st>>>(w, C, Cout, dg, N, nch, nkp,
                                                                reinterpret_cast<uint8_t *>(packed));
    C2M_LAUNCH_CHECK("dcn_dgrad_wpack_kernel");
    return C2M_OK;
}

template <int N>
static void launch_dgrad(bool gi, int grid, cudaStream_t st, const CUtensorMap &mh, const CUtensorMap &ml,
                         const DcnGrad &d) {
    if (gi) {
        cudaFuncSetAttribute(dcn_dgrad_kernel<N, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DG_SMEM);
        dcn_dgrad_kernel<N, true><<<grid, DG_THREADS, DG_SMEM, st>>>(mh, ml, d);
    } else {
        cudaFuncSetAttribute(dcn_dgrad_kernel<N, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DG_SMEM);
        dcn_dgrad_kernel<N, false><<<grid, DG_THREADS, DG_SMEM, st>>>(mh, ml, d);
    }
}

extern "C" int c2m_dcn_tc_dgrad(const c2m_dcn_tc_grad_args *a, c2m_stream_t stream) {
    if (const int rc = check_grad_args(a, "dcn_tc_dgrad")) return rc;
    C2M_CHECK_ARG(a->packed_w && a->grad_offset && a->grad_mask, "dcn_tc_dgrad: null pointer");
    DcnGrad d;
    grad_geom(a->B, a->C, a->H, a->W, a->Cout, a->dg, d);
    d.x_il = reinterpret_cast<const __half *>(a->x_il);
    d.x_amax = a->x_amax; d.mask_amax = a->mask_amax; d.gy_amax = a->gy_amax;
    d.off = a->offset; d.mask = a->mask;
    d.wblob = reinterpret_cast<const uint8_t *>(a->packed_w);
    d.goff = a->grad_offset; d.gmask = a->grad_mask; d.gx = a->grad_input;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CUtensorMap mh, ml;
    int rc;
    if ((rc = make_psa_tensor_map(&mh, a->gy_hi, a->B, d.C8o, a->H, a->W, T_C, T_R))) return rc;
    if ((rc = make_psa_tensor_map(&ml, a->gy_lo, a->B, d.C8o, a->H, a->W, T_C, T_R))) return rc;
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    const int grid = d.ntiles < sms ? (int)d.ntiles : sms;
    const double px = (double)a->B * a->H * a->W;
    void *ph = prof_begin(PROF_DCN_DGRAD, 2.0 * a->Cout * a->C * 9.0 * px,
                          4.0 * px * (a->Cout + 27.0 * a->dg + a->C * (a->grad_input ? 2.0 : 1.0)), st);
    const bool gi = a->grad_input != nullptr;
    switch (d.N) {
    case 8: launch_dgrad<8>(gi, grid, st, mh, ml, d); break;
    case 16: launch_dgrad<16>(gi, grid, st, mh, ml, d); break;
    case 24: launch_dgrad<24>(gi, grid, st, mh, ml, d); break;
    case 32: launch_dgrad<32>(gi, grid, st, mh, ml, d); break;
    case 40: launch_dgrad<40>(gi, grid, st, mh, ml, d); break;
    case 48: launch_dgrad<48>(gi, grid, st, mh, ml, d); break;
    case 56: launch_dgrad<56>(gi, grid, st, mh, ml, d); break;
    default: launch_dgrad<64>(gi, grid, st, mh, ml, d); break;
    }
    C2M_LAUNCH_CHECK("dcn_dgrad_kernel");
    prof_end(ph, st);
    return C2M_OK;
}

extern "C" size_t c2m_dcn_tc_wgrad_workspace_bytes(int B, int C, int H, int W, int Cout, int dg) {
    if (B <= 0 || H <= 0 || W <= 0 || !c2m_dcn_tc_supported(C, Cout, dg)) {
        set_error("dcn_tc_wgrad_workspace_bytes: bad shape");
        return 0;
    }
    DcnGrad d;
    grad_geom(B, C, H, W, Cout, dg, d);
    if (wgrad_ksplit(d.nkc * d.ncs, d.ntiles, d.ksplit)) return 0;
    return wgrad_ws_bytes(d.ksplit, d.ncs * WG_NCO, d.nkc * 32);
}

extern "C" int c2m_dcn_tc_wgrad(const c2m_dcn_tc_grad_args *a, c2m_stream_t stream) {
    if (const int rc = check_grad_args(a, "dcn_tc_wgrad")) return rc;
    C2M_CHECK_ARG(a->grad_weight, "dcn_tc_wgrad: null pointer");
    DcnGrad d;
    grad_geom(a->B, a->C, a->H, a->W, a->Cout, a->dg, d);
    if (const int rc = wgrad_ksplit(d.nkc * d.ncs, d.ntiles, d.ksplit)) return rc;
    const size_t need = wgrad_ws_bytes(d.ksplit, d.ncs * WG_NCO, d.nkc * 32);
    if (!a->ws || a->ws_bytes < need) {
        set_error("dcn_tc_wgrad: workspace of %zu bytes, %zu needed", a->ws_bytes, need);
        return C2M_ERR_WORKSPACE;
    }
    d.x_il = reinterpret_cast<const __half *>(a->x_il);
    d.x_amax = a->x_amax; d.mask_amax = a->mask_amax; d.gy_amax = a->gy_amax;
    d.off = a->offset; d.mask = a->mask;
    d.ws = reinterpret_cast<float *>(a->ws);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CUtensorMap mh, ml;
    int rc;
    if ((rc = make_psa_tensor_map(&mh, a->gy_hi, a->B, d.C8o, a->H, a->W, T_C, T_R))) return rc;
    if ((rc = make_psa_tensor_map(&ml, a->gy_lo, a->B, d.C8o, a->H, a->W, T_C, T_R))) return rc;
    const int grid = d.nkc * d.ncs * d.ksplit;
    const double px = (double)a->B * a->H * a->W;
    void *ph = prof_begin(PROF_DCN_WGRAD, 2.0 * a->Cout * a->C * 9.0 * px,
                          4.0 * px * (a->Cout + 27.0 * a->dg + a->C), st);
    if (d.nh == 1) {
        const size_t smem = (size_t)WG_NSY * 2 * 8 * OCT_B + WG_NSG * WG_COL_STAGE + (2 * WG_NSY + 2 * WG_NSG) * 8 + 1024;
        C2M_CUDA(cudaFuncSetAttribute(dcn_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dcn_wgrad_kernel<1><<<grid, NTHREADS, smem, st>>>(mh, ml, d);
    } else {
        const size_t smem = (size_t)WG_NSY * 2 * 16 * OCT_B + WG_NSG * WG_COL_STAGE + (2 * WG_NSY + 2 * WG_NSG) * 8 + 1024;
        C2M_CUDA(cudaFuncSetAttribute(dcn_wgrad_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dcn_wgrad_kernel<2><<<grid, NTHREADS, smem, st>>>(mh, ml, d);
    }
    C2M_LAUNCH_CHECK("dcn_wgrad_kernel");
    wgrad_reduce_kernel<<<grid_blocks((long long)a->Cout * d.nkc * 32), 256, 0, st>>>(
        d.ws, d.ksplit, a->C, a->Cout, d.cpg, d.ncs * WG_NCO, d.nkc * 32, a->grad_weight);
    C2M_LAUNCH_CHECK("wgrad_reduce_kernel");
    prof_end(ph, st);
    return C2M_OK;
}
