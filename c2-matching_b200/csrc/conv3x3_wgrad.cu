// Backward of the 3x3 / stride 1 / pad 1 convolution: gradient scaling on the device and the weight gradient on the
// sm_90a tensor cores (wgmma), fp32-grade (split fp16 x 3, as the forward in conv3x3_umma.cu).
//
// The input gradient needs no kernel of its own: dX is the 3x3 convolution of grad_output with the weights transposed
// in Cin / Cout and rotated by 180 degrees, so it runs on conv3x3_wgmma_kernel with a second packed weight blob.
//
// Loss gradients are tiny (an L1 mean over a 9 x 3 x 160 x 160 batch gives ~2^-19 per element) and would lose their lo
// halves to fp16 subnormals at scale exponent 0.  grad_output therefore enters as the forward's x does
// (c2m_conv3x3_operand_f32): image b is stored as grad_output * 2^sg_b, sg_b = 14 - exponent(largest finite |grad_output|
// of image b), computed on the device.  The results divide 2^sg_b back out on the device, image by image, so no host
// synchronisation is needed, an image's gradients do not depend on the other images' magnitudes, and grad_output * 2^k
// gives exactly 2^k times the gradients.
//
// Weight gradient, dW[co][ci][tap] = sum over (b, y, x) of gY[b,co,y,x] * X[b,ci,(y,x) + delta_tap]: a GEMM with
// M = Cout, N = Cin x 9 taps and K = every pixel of the batch.  Both operands are PSA tensors, fp16 [B][C/8][H][W][8]:
// 8 channels of one pixel are 16 contiguous bytes, so along K = pixels they are MN-major (transposed) wgmma operands,
// and 8 consecutive pixels of one octet plane are one 128-byte core matrix.  A CTA computes a 64-wide Cout slice x a
// 32-wide Cin chunk x 9 taps over a contiguous range of 16x8-pixel tiles: per tile, one TMA box of gY (16 x 8 pixels,
// 8 octets) and one halo'd box of X (18 x 10 pixels, 4 octets) per half; two 8-pixel tile rows (two core matrices
// along K) are one K=16 step, and a tap's shifted X view is the same descriptor moved by (dy * 10 + dx) * 16 bytes.
// Three products per step: hi*hi + hi*lo + lo*hi.  The two consumer warpgroups split the taps; the CTA writes its
// 64 x 32 x 9 fp32 partial to its own workspace slot, and c2m_conv3x3_wgrad then sums the slots in one fixed order, so
// dW is the same bit for bit on every run on a given device.
#include "umma_conv_common.cuh"

namespace c2m {

namespace {
constexpr int G_R = 16, G_C = 8;                 // gY tile: 16 rows x 8 pixels (two rows = one K=16 step)
constexpr int X_R = G_R + 2, X_C = G_C + 2;      // halo'd X tile (the forward's 18 x 10 box)
constexpr int G_OCT = 8, X_OCT = 4;              // 64 output channels x 32 input channels per CTA
constexpr int G_ROW_B = G_C * 16;                // 128 B
constexpr int G_OCT_B = G_R * G_ROW_B;           // 2048 B
constexpr int G_HALF = G_OCT * G_OCT_B;          // 16384 B
constexpr int X_ROW_B = X_C * 16;                // 160 B
constexpr int X_OCT_B = X_R * X_ROW_B;           // 2880 B
constexpr int X_HALF = X_OCT * X_OCT_B;          // 11520 B
constexpr int WG_STAGE = 2 * G_HALF + 2 * X_HALF;   // 55808 B
constexpr int WG_NST = 3;
constexpr size_t WG_SMEM = (size_t)WG_NST * WG_STAGE + 2 * WG_NST * 8 + 1024;
constexpr int WG_CO = G_OCT * 8, WG_CI = X_OCT * 8;
constexpr int WG_FLUSH = 8;                      // tiles (8 x 8 K steps x 3 MMAs) per accumulator run

struct WgradGeom {
    int B, H, W, Cin, Cout, C8i, C8o;
    int nslice, nchunk, ksplit;
    int tiles_x, tiles_y;
    long long ntiles;
    const unsigned *gy_amax;    // [B]: image b of gY is stored as gy * 2^grad_scale_exp(gy_amax + b)
    const unsigned *x_amax;     // [B] or null: image b of X is stored as x * 2^grad_scale_exp(x_amax + b)
};

// Tile t of the batch: image b and top-left pixel (y0, x0).  The last tile row and column are moved back inside the
// map (y0 = H - 16, x0 = W - 8) when the map is not a multiple of the tile, so no tile holds a pixel outside the map:
// a zero-filled grad_output there would meet X's last row or column at tap ky = 0 / kx = 0, and 0 * Inf is NaN.  The
// first dy rows and dx columns of such a tile were already summed by its neighbour; the consumers zero them in gY.
struct WgradTile { int b, y0, x0, dy, dx; };
__device__ __forceinline__ WgradTile wgrad_tile(const WgradGeom &p, long long t) {
    const int tiles_img = p.tiles_x * p.tiles_y;
    WgradTile r;
    r.b = (int)(t / tiles_img);
    const int tt = (int)(t % tiles_img);
    r.y0 = (tt / p.tiles_x) * G_R;
    r.x0 = (tt % p.tiles_x) * G_C;
    r.dy = max(0, r.y0 + G_R - p.H);
    r.dx = max(0, r.x0 + G_C - p.W);
    r.y0 -= r.dy;
    r.x0 -= r.dx;
    return r;
}
}  // namespace

__global__ void grad_amax_kernel(const float *__restrict__ g, int C, int H, int W, long long s_b, long long s_c,
                                 long long s_y, long long s_x, unsigned *__restrict__ amax, int amax_step) {
    const long long n = (long long)C * H * W;
    const int b = blockIdx.y;
    float m = 0.f;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(e / ((long long)H * W));
        const long long pix = e % ((long long)H * W);
        const float a = fabsf(g[b * s_b + c * s_c + (pix / W) * s_y + (pix % W) * s_x]);
        if (a < INFINITY) m = fmaxf(m, a);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax + b * amax_step, __float_as_uint(m));
}

// Consumer warpgroup of conv3x3_wgrad_kernel: taps [T0, T0 + NT) of every K step of tiles [t0, t1), then the 64 x 32 x NT
// partial into the CTA's workspace slot `dst` ([co_pad][tap][ci_pad] fp32, see wgrad_flush).
template <int T0, int NT>
__device__ __forceinline__ void wgrad_consume(uint8_t *smem, uint64_t *full, uint64_t *empty, long long t0, long long t1,
                                              const WgradGeom &p, int slice, int chunk, float *dst) {
    float acc[NT][16];
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[t][i] = 0.f;
    const int ci_pad = p.nchunk * WG_CI, ncol = 9 * ci_pad;
    float *blk = dst + (size_t)slice * WG_CO * ncol + T0 * ci_pad + chunk * WG_CI;
    bool first = true;
    // each accumulator run holds one image: the flush divides its two operand exponents back out (their sum can reach
    // +-240, see wgrad_flush)
    auto flush = [&](int b) {
        const int e = b < 0 ? 0 : -(grad_scale_exp(p.gy_amax + b) + (p.x_amax ? grad_scale_exp(p.x_amax + b) : 0));
        wgrad_flush(acc, blk, ncol, ci_pad, first, e);
        first = false;
    };
    int stage = 0, phase = 0, n = 0, cur_b = -1;
    for (long long t = t0; t < t1; ++t) {
        const WgradTile tl = wgrad_tile(p, t);
        if (n > 0 && (tl.b != cur_b || n == WG_FLUSH)) { flush(cur_b); n = 0; }
        cur_b = tl.b;
        mbar_wait(&full[stage], phase);
        const uint32_t s = smem_u32(smem + stage * WG_STAGE);
        if (tl.dy | tl.dx) {
            // a tile moved back inside the map: zero gY (both halves, every octet) at the rows / columns its
            // neighbour already summed, then make the writes visible to the tensor cores of both warpgroups
            uint4 *g = reinterpret_cast<uint4 *>(smem + stage * WG_STAGE);
            for (int i = threadIdx.x - 128; i < 2 * G_OCT * G_R * G_C; i += 256) {
                const int c = i % G_C, r = (i / G_C) % G_R;
                if (r < tl.dy || c < tl.dx) g[i] = make_uint4(0, 0, 0, 0);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("bar.sync 1, 256;" ::: "memory");
        }
        // MN-major descriptors: lbo = next core matrix along K (the next tile row), sbo = next octet along M / N.
        // A = gY (M = Cout, K = pixels), B = X (N = Cin, K = pixels).
        const uint64_t dgh = wg_smem_desc(s, G_ROW_B, G_OCT_B), dgl = wg_smem_desc(s + G_HALF, G_ROW_B, G_OCT_B);
        const uint64_t dxh = wg_smem_desc(s + 2 * G_HALF, X_ROW_B, X_OCT_B);
        const uint64_t dxl = wg_smem_desc(s + 2 * G_HALF + X_HALF, X_ROW_B, X_OCT_B);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < G_R / 2; ++j) {              // K step j: tile rows 2j and 2j + 1
            const uint32_t ga = 2 * j * G_ROW_B;
#pragma unroll
            for (int tt = 0; tt < NT; ++tt) {
                const int tap = T0 + tt;
                const uint32_t xb = (2 * j + tap / 3) * X_ROW_B + (tap % 3) * 16;
                wgmma_tt_split(acc[tt], wg_desc_advance(dgh, ga), wg_desc_advance(dgl, ga), wg_desc_advance(dxh, xb),
                               wg_desc_advance(dxl, xb));
            }
        }
        wgmma_commit();
        wgmma_wait_all();
        mbar_arrive(&empty[stage]);
        if (++stage == WG_NST) { stage = 0; phase ^= 1; }
        ++n;
    }
    if (n || first) flush(cur_b);
}

// ------------------------------------------------------------------------------------------
// CTA (slice, chunk, k) = blockIdx.x decomposed slice-fastest: the CTAs of one K range are neighbours and read the same
// tiles together.  Warp 0 of warpgroup 0 streams the tiles through a WG_NST-deep TMA ring; warpgroups 1 and 2 consume
// them (wgrad_consume) and write their taps of the CTA's partial to workspace slot k.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(384, 1)
conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap tg_hi, const __grid_constant__ CUtensorMap tg_lo,
                     const __grid_constant__ CUtensorMap tx_hi, const __grid_constant__ CUtensorMap tx_lo,
                     const WgradGeom p, float *__restrict__ ws) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + WG_NST * WG_STAGE), *empty = full + WG_NST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slice = blockIdx.x % p.nslice;
    const int chunk = (blockIdx.x / p.nslice) % p.nchunk;
    const int k = blockIdx.x / (p.nslice * p.nchunk);
    const long long t0 = p.ntiles * k / p.ksplit, t1 = p.ntiles * (k + 1) / p.ksplit;
    // the second gY box (octets 4..7 of the slice) holds only zero padding when the slice has <= 32 channels: skip it
    const bool g_second = slice * G_OCT + 4 < p.C8o;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tg_hi);
        tma_prefetch_desc(&tg_lo);
        tma_prefetch_desc(&tx_hi);
        tma_prefetch_desc(&tx_lo);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < WG_NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            const uint32_t bytes = 2 * (g_second ? G_HALF : G_HALF / 2) + 2 * X_HALF;
            int stage = 0, phase = 0;
            for (long long t = t0; t < t1; ++t) {
                const WgradTile tl = wgrad_tile(p, t);
                const int b = tl.b, y0 = tl.y0, x0 = tl.x0;
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t *s = smem + stage * WG_STAGE;
                mbar_arrive_expect_tx(&full[stage], bytes);
                tma_load_4d(s, &tg_hi, &full[stage], x0 * 8, y0, slice * G_OCT, b);
                tma_load_4d(s + G_HALF, &tg_lo, &full[stage], x0 * 8, y0, slice * G_OCT, b);
                if (g_second) {
                    tma_load_4d(s + G_HALF / 2, &tg_hi, &full[stage], x0 * 8, y0, slice * G_OCT + 4, b);
                    tma_load_4d(s + G_HALF + G_HALF / 2, &tg_lo, &full[stage], x0 * 8, y0, slice * G_OCT + 4, b);
                }
                tma_load_4d(s + 2 * G_HALF, &tx_hi, &full[stage], (x0 - 1) * 8, y0 - 1, chunk * X_OCT, b);
                tma_load_4d(s + 2 * G_HALF + X_HALF, &tx_lo, &full[stage], (x0 - 1) * 8, y0 - 1, chunk * X_OCT, b);
                if (++stage == WG_NST) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // warpgroup 1 takes taps 0..4, warpgroup 2 taps 5..8 (80 / 64 accumulator registers: the kernel's register
        // budget of 168 per thread does not hold all nine 64 x 32 tiles in one warpgroup)
        float *slot = ws + (size_t)k * p.nslice * WG_CO * 9 * p.nchunk * WG_CI;
        if (warp < 8) wgrad_consume<0, 5>(smem, full, empty, t0, t1, p, slice, chunk, slot);
        else wgrad_consume<5, 4>(smem, full, empty, t0, t1, p, slice, chunk, slot);
    }
}

__global__ void wgrad_reduce_kernel(const float *__restrict__ ws, int nslots, int C, int Cout, int cpg, int co_pad,
                                    int ncol, float *__restrict__ dw) {
    const long long n = (long long)Cout * ncol;
    const size_t slot = (size_t)co_pad * ncol;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(e / ncol), col = (int)(e % ncol);
        const int pair = col / cpg, c = (pair / 9) * cpg + col % cpg;     // pair = (group, tap)
        if (c >= C) continue;                                             // padding column
        float v = 0.f;
        for (int j = 0; j < nslots; ++j) v += ws[e + j * slot];
        dw[((size_t)co * C + c) * 9 + pair % 9] = v;
    }
}

static int wgrad_geom(int B, int Cin, int Cout, int H, int W, WgradGeom &g) {
    g.B = B; g.H = H; g.W = W; g.Cin = Cin; g.Cout = Cout;
    g.gy_amax = g.x_amax = nullptr;
    g.C8i = (Cin + 7) / 8; g.C8o = (Cout + 7) / 8;
    g.nslice = ceil_div(Cout, WG_CO);
    g.nchunk = ceil_div(Cin, WG_CI);
    g.tiles_x = ceil_div(W, G_C);
    g.tiles_y = ceil_div(H, G_R);
    g.ntiles = (long long)B * g.tiles_x * g.tiles_y;
    return wgrad_ksplit(g.nslice * g.nchunk, g.ntiles, g.ksplit);
}

}  // namespace c2m

using namespace c2m;

extern "C" int c2m_conv3x3_operand_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c,
                                       long long xs_y, long long xs_x, void *hi, void *lo, unsigned *amax,
                                       c2m_stream_t stream) {
    C2M_CHECK_ARG(x && hi && lo && amax && B > 0 && C > 0 && H > 0 && W > 0, "conv3x3_operand_f32: bad argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    C2M_CUDA(cudaMemsetAsync(amax, 0, B * sizeof(unsigned), st));
    const long long n = (long long)C * H * W;
    const int ba = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    grad_amax_kernel<<<dim3(ba, B), 256, 0, st>>>(x, C, H, W, xs_b, xs_c, xs_y, xs_x, amax, 1);
    C2M_LAUNCH_CHECK("grad_amax_kernel");
    const int C8 = (C + 7) / 8;
    const long long np = (long long)C8 * H * W;
    const int bx = (int)((np + 255) / 256 < 4096 ? (np + 255) / 256 : 4096);
    psa_from_f32_kernel<<<dim3(bx, B), 256, 0, st>>>(x, C, C8, H, W, xs_b, xs_c, xs_y, xs_x, 0, amax,
                                                     reinterpret_cast<__half *>(hi), reinterpret_cast<__half *>(lo));
    C2M_LAUNCH_CHECK("psa_from_f32_kernel");
    return C2M_OK;
}

extern "C" size_t c2m_conv3x3_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W) {
    if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) {
        set_error("conv3x3_wgrad_workspace_bytes: bad shape");
        return 0;
    }
    WgradGeom g;
    if (wgrad_geom(B, Cin, Cout, H, W, g)) return 0;
    return wgrad_ws_bytes(g.ksplit, g.nslice * WG_CO, 9 * g.nchunk * WG_CI);
}

// x_amax null: X is PSA at scale exponent 0
static int conv3x3_wgrad(const void *gy_hi, const void *gy_lo, const unsigned *gy_amax, const void *x_hi,
                         const void *x_lo, const unsigned *x_amax, int B, int Cin, int Cout, int H, int W, float *dw,
                         void *ws, size_t ws_bytes, c2m_stream_t stream) {
    C2M_CHECK_ARG(gy_hi && gy_lo && gy_amax && x_hi && x_lo && dw, "conv3x3_wgrad: null pointer");
    C2M_CHECK_ARG(B > 0 && Cin > 0 && Cout > 0, "conv3x3_wgrad: bad shape");
    C2M_CHECK_ARG(H >= X_R && W >= X_C, "conv3x3_wgrad: map %dx%d smaller than one halo tile (18x10)", H, W);
    WgradGeom g;
    if (const int rc = wgrad_geom(B, Cin, Cout, H, W, g)) return rc;
    g.gy_amax = gy_amax;
    g.x_amax = x_amax;
    const int co_pad = g.nslice * WG_CO, ci_pad = g.nchunk * WG_CI;
    const size_t need = wgrad_ws_bytes(g.ksplit, co_pad, 9 * ci_pad);
    if (!ws || ws_bytes < need) {
        set_error("conv3x3_wgrad: workspace of %zu bytes, %zu needed", ws_bytes, need);
        return C2M_ERR_WORKSPACE;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CUtensorMap mgh, mgl, mxh, mxl;
    int rc;
    if ((rc = make_psa_tensor_map(&mgh, gy_hi, B, g.C8o, H, W, G_C, G_R))) return rc;
    if ((rc = make_psa_tensor_map(&mgl, gy_lo, B, g.C8o, H, W, G_C, G_R))) return rc;
    if ((rc = make_psa_tensor_map(&mxh, x_hi, B, g.C8i, H, W, X_C, X_R))) return rc;
    if ((rc = make_psa_tensor_map(&mxl, x_lo, B, g.C8i, H, W, X_C, X_R))) return rc;
    C2M_CUDA(cudaFuncSetAttribute(conv3x3_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM));
    const int grid = g.nslice * g.nchunk * g.ksplit;
    float *part = reinterpret_cast<float *>(ws);
    // algorithmic work: 2 * Cin * Cout * 9 flops per pixel; bytes = the two PSA operands (4 B / element) + dW
    const double px = (double)B * H * W;
    void *ph = prof_begin(PROF_CONV3X3_WGRAD, 2.0 * Cin * Cout * 9.0 * px, 4.0 * px * (Cin + Cout) + 36.0 * Cin * Cout,
                          st);
    conv3x3_wgrad_kernel<<<grid, 384, WG_SMEM, st>>>(mgh, mgl, mxh, mxl, g, part);
    C2M_LAUNCH_CHECK("conv3x3_wgrad_kernel");
    prof_end(ph, st);
    wgrad_reduce_kernel<<<grid_blocks((long long)Cout * 9 * ci_pad), 256, 0, st>>>(part, g.ksplit, Cin, Cout, ci_pad,
                                                                                co_pad, 9 * ci_pad, dw);
    C2M_LAUNCH_CHECK("wgrad_reduce_kernel");
    return C2M_OK;
}

extern "C" int c2m_conv3x3_wgrad(const void *gy_hi, const void *gy_lo, const unsigned *gy_amax, const void *x_hi,
                                 const void *x_lo, int B, int Cin, int Cout, int H, int W, float *dw, void *ws,
                                 size_t ws_bytes, c2m_stream_t stream) {
    return conv3x3_wgrad(gy_hi, gy_lo, gy_amax, x_hi, x_lo, nullptr, B, Cin, Cout, H, W, dw, ws, ws_bytes, stream);
}

extern "C" int c2m_conv3x3_wgrad_scaled(const void *gy_hi, const void *gy_lo, const unsigned *gy_amax,
                                        const void *x_hi, const void *x_lo, const unsigned *x_amax, int B, int Cin,
                                        int Cout, int H, int W, float *dw, void *ws, size_t ws_bytes,
                                        c2m_stream_t stream) {
    C2M_CHECK_ARG(x_amax, "conv3x3_wgrad_scaled: null x_amax");
    return conv3x3_wgrad(gy_hi, gy_lo, gy_amax, x_hi, x_lo, x_amax, B, Cin, Cout, H, W, dw, ws, ws_bytes, stream);
}
