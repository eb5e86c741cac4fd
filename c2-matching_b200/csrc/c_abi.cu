// C-ABI entry points of libc2m_sm100 that are not defined next to their kernel: error/launch
// bookkeeping and the correlation driver (workspace carving + prep -> search -> rescore).
#include <atomic>
#include <cstdarg>
#include <cstring>
#include <mutex>
#include <vector>

#include "corr_internal.cuh"

namespace c2m {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_psa_tensor_map(CUtensorMap *map, const void *base, int B, int C8, int H, int W, int box_px, int box_rows) {
    static EncodeTiledFn enc = nullptr;
    if (!enc) {
        void *pfn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &pfn, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point not available");
            return C2M_ERR_UNSUPPORTED;
        }
        enc = reinterpret_cast<EncodeTiledFn>(pfn);
    }
    cuuint64_t dims[4] = {(cuuint64_t)W * 8, (cuuint64_t)H, (cuuint64_t)C8, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)C8 * H * W * 16};
    cuuint32_t box[4] = {(cuuint32_t)box_px * 8, (cuuint32_t)box_rows, 4, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return C2M_ERR_CUDA; }
    return C2M_OK;
}

static std::atomic<int> g_profile{0};
static std::mutex g_prof_mu;
struct ProfRec { int kernel; double flops, bytes; cudaEvent_t e0, e1; };
static std::vector<ProfRec *> g_prof_recs;

bool prof_enabled() { return g_profile.load() != 0; }

void *prof_begin(int kernel, double flops, double bytes, cudaStream_t st) {
    if (!prof_enabled()) return nullptr;
    ProfRec *r = new ProfRec{kernel, flops, bytes, nullptr, nullptr};
    if (cudaEventCreate(&r->e0) != cudaSuccess || cudaEventCreate(&r->e1) != cudaSuccess ||
        cudaEventRecord(r->e0, st) != cudaSuccess) {
        delete r;
        return nullptr;
    }
    return r;
}

void prof_end(void *handle, cudaStream_t st) {
    if (!handle) return;
    ProfRec *r = static_cast<ProfRec *>(handle);
    cudaEventRecord(r->e1, st);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_recs.push_back(r);
}

static int make_geom(CorrGeom &g, int B, int C, int h, int w, int hr, int wr, int patch, int s_in, int s_ref) {
    C2M_CHECK_ARG(B > 0 && C > 0, "corr: empty batch or channels (B=%d C=%d)", B, C);
    C2M_CHECK_ARG(patch > 0 && s_in > 0 && s_ref > 0, "corr: bad patch/stride");
    C2M_CHECK_ARG(h >= patch && w >= patch && hr >= patch && wr >= patch,
                  "corr: map smaller than the patch (in %dx%d, ref %dx%d, patch %d)", h, w, hr, wr, patch);
    g.B = B; g.C = C; g.Cp = (C + 7) / 8 * 8;
    g.h = h; g.w = w; g.hr = hr; g.wr = wr;
    g.patch = patch; g.s_in = s_in; g.s_ref = s_ref;
    g.gh = (h - patch) / s_in + 1; g.gw = (w - patch) / s_in + 1;
    g.rh = (hr - patch) / s_ref + 1; g.rw = (wr - patch) / s_ref + 1;
    g.NQ = g.gh * g.gw; g.NR = g.rh * g.rw;
    return C2M_OK;
}

// carve the caller's workspace; with base == nullptr only sizes are computed
static void carve(CorrWorkspace &ws, const CorrGeom &g, uint8_t *base) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t *p = base ? base + off : nullptr;
        off += align_up(bytes, 256);
        return p;
    };
    const size_t pin = (size_t)g.B * g.h * g.w, pref = (size_t)g.B * g.hr * g.wr;
    ws.p32_in = (float *)take(pin * g.Cp * 4);
    ws.p32_ref = (float *)take(pref * g.Cp * 4);
    ws.hi_in = (__half *)take(pin * g.Cp * 2);
    ws.lo_in = (__half *)take(pin * g.Cp * 2);
    ws.hi_ref = (__half *)take(pref * g.Cp * 2);
    ws.lo_ref = (__half *)take(pref * g.Cp * 2);
    ws.ss_in = (float *)take(pin * 4);
    ws.ss_ref = (float *)take(pref * 4);
    ws.rinv = (float *)take((size_t)g.B * g.NR * 4);
    ws.part = (Candidate *)take((size_t)g.B * CORR_MAX_CHUNKS * g.NQ * sizeof(Candidate));
    ws.ovf = (CorrOverflow *)take((size_t)g.B * g.NQ * sizeof(CorrOverflow));
    ws.best = (unsigned long long *)take((size_t)g.B * g.NQ * 8);
    ws.qnorm = (float *)take((size_t)g.B * g.NQ * 4);
    ws.amax_bits = (unsigned *)take(256);            // zeroed at the start of every call
    ws.sexp = (int *)(ws.amax_bits ? ws.amax_bits + 8 : nullptr);
    ws.ovf_count = ws.amax_bits ? ws.amax_bits + 16 : nullptr;
    ws.max_pn_bits = ws.amax_bits ? ws.amax_bits + 17 : nullptr;
    ws.rinv_max_bits = ws.amax_bits ? ws.amax_bits + 18 : nullptr;
    ws.total_bytes = off;
}

}  // namespace c2m

using namespace c2m;

// 7: gy_amax is [B] (one grad_output exponent per image), no c2m_grad_psa_from_f32 / c2m_grad_unscale_f32; 6: no fp32
// c2m_dcn_v2_* twins of c2m_deform_conv_*; 5: c2m_dcn_tc_args without x_hi / x_lo; 4: .x_il +
// c2m_psa_interleave; 3: .mask; 2: out_f32_octets / om_octets.  (c2m_dcn_tc_args has since gained x_amax / mask_amax at
// its end and c2m_psa_interleave became c2m_dcn_tc_operand_psa; c2m_conv3x3_args gained x_amax at its end, with
// c2m_conv3x3_operand_f32 and c2m_conv3x3_wgrad_scaled: the bindings resolve every declared symbol, so a library older
// than those fails to load.)
extern "C" int c2m_abi_version(void) { return 7; }
extern "C" const char *c2m_last_error(void) { return g_err; }
extern "C" unsigned long long c2m_launch_count(void) { return g_launches.load(); }

extern "C" size_t c2m_corr_workspace_bytes(int B, int C, int h, int w, int hr, int wr, int patch, int s_in, int s_ref) {
    CorrGeom g;
    if (make_geom(g, B, C, h, w, hr, wr, patch, s_in, s_ref)) return 0;
    CorrWorkspace ws;
    carve(ws, g, nullptr);
    return ws.total_bytes;
}

extern "C" int c2m_corr_argmax_f32(const float *fin, const float *fref, int B, int C, int h, int w, int hr, int wr,
                                   int patch, int s_in, int s_ref, int is_norm, int norm_input, int l2norm,
                                   unsigned flags, int64_t *idx, float *val, void *wsp, size_t ws_bytes,
                                   c2m_stream_t stream) {
    C2M_CHECK_ARG(fin && fref && idx && val, "corr_argmax: null pointer");
    CorrGeom g;
    int rc = make_geom(g, B, C, h, w, hr, wr, patch, s_in, s_ref);
    if (rc) return rc;
    CorrWorkspace ws;
    carve(ws, g, reinterpret_cast<uint8_t *>(wsp));
    if (!wsp || ws_bytes < ws.total_bytes) {
        set_error("corr_argmax: workspace of %zu bytes given, %zu needed", ws_bytes, ws.total_bytes);
        return C2M_ERR_WORKSPACE;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    C2M_CUDA(cudaMemsetAsync(ws.amax_bits, 0, 256, st));

    const bool use_umma = !(flags & 1u) && corr_umma_supported(g);
    CorrChunkGeom cg;
    float window_coef, sub_coef = 0.f;
    const int K = g.C * g.patch * g.patch;
    int sms = 0;
    C2M_CUDA(sm_count(sms));
    if (use_umma) {
        int dev = 0, major = 0;
        C2M_CUDA(cudaGetDevice(&dev));
        C2M_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
        if (major != 9) {
            set_error("corr_argmax: wgmma path needs an sm_90 device (found sm_%d*)", major);
            return C2M_ERR_UNSUPPORTED;
        }
        ws.nchunk = corr_umma_pick_nchunk(g, sms);
        corr_umma_chunk_geom(g, ws.nchunk, cg);
        // DESIGN.md K2: the search scores (q_hi + q_lo) . r_hi.  |approx - exact| <= E = [2^-11 + 2^-22 (K/16 + 3)] ||P_q||
        // ||P_r|| rinv_r + E_sub: 2^-11 = fp16 rounding of the Ref operand (Cauchy-Schwarz over the patch), K/16 wgmma
        // instructions feed each score with 1 fp32 ulp of (|acc| + sum|products|) each, + the query's 2^-22 split.
        // Window = 2E for the rounding part (best and candidate both err; 1 % margin) and 4E for the accumulation part
        // (x2 of slack for the tensor core's internal alignment).
        // E_sub: one scale exponent per map and call (|x| 2^sexp <= 1024 for the largest |x| of the whole batch) puts
        // elements far below that maximum into the fp16 subnormals, whose rounding is absolute: up to 2^-25 per element
        // of r_hi and of q_hi + q_lo, i.e. sqrt(K) 2^-25 over a patch.  E_sub = sqrt(K) 2^-25 [2^-sexp_in ||P_r|| rinv_r
        // + ||P_q|| 2^-sexp_ref rinv_r], with ||P_r|| rinv_r <= 1 (max ||P_r|| for raw scores) and rinv_r <= the largest
        // rinv of a nonzero Ref patch (an all-zero patch rounds exactly).  With l2norm (sexp = 10, pixel norms 1 or 0)
        // it is ~1e-6 of the window.
        window_coef = 1.01f * ldexpf(1.f, -10) + ldexpf(1.f, -20) * (float)((K + 15) / 16 + 3);
        sub_coef = 1.01f * ldexpf(1.f, -24) * sqrtf((float)(g.Cp * g.patch * g.patch));
    } else {
        int n = ceil_div(4 * sms, g.B * ceil_div(g.NQ, 64));
        const int ntile = ceil_div(g.NR, 64);
        if (n > CORR_MAX_CHUNKS) n = CORR_MAX_CHUNKS;
        if (n > ntile) n = ntile;
        if (n < 1) n = 1;
        ws.nchunk = n;
        corr_generic_chunk_geom(g, ws.nchunk, cg);
        // sequential fp32 FMA chain of K terms: |approx - exact| <= K * 2^-24 * ||P_q|| * ||P_r|| * rinv_r (+ the final scale)
        window_coef = ldexpf(1.f, -23) * (float)(K + 4);
    }

    if ((rc = corr_prep_launch(fin, B, C, g.Cp, h * w, l2norm, 0, ws, ws.p32_in, ws.hi_in, ws.lo_in, ws.ss_in, st))) return rc;
    if ((rc = corr_prep_launch(fref, B, C, g.Cp, hr * wr, l2norm, 1, ws, ws.p32_ref, ws.hi_ref, ws.lo_ref, ws.ss_ref, st))) return rc;
    if ((rc = corr_rinv_launch(g, ws, is_norm, st))) return rc;
    const double flops = 2.0 * g.C * g.patch * g.patch * (double)g.NQ * g.NR * g.B;
    const double bytes = (4.0 * g.C * ((double)g.h * g.w + (double)g.hr * g.wr) + 12.0 * g.NQ) * g.B;
    void *ph = prof_begin(PROF_CORR_SEARCH, flops, bytes, st);
    rc = use_umma ? corr_search_umma_launch(g, ws, st) : corr_search_generic_launch(g, ws, st);
    if (rc) return rc;
    prof_end(ph, st);
    return corr_rescore_launch(g, ws, cg, window_coef, sub_coef, is_norm, norm_input, idx, val, st);
}

extern "C" int c2m_profile_enable(int on) {
    g_profile.store(on ? 1 : 0);
    return C2M_OK;
}

extern "C" int c2m_profile_collect(int kernel, float *ms_total, int *launches, double *flops, double *bytes) {
    C2M_CHECK_ARG(ms_total && launches && flops && bytes && kernel >= 0 && kernel < PROF_NKERNELS, "profile_collect: bad argument");
    std::lock_guard<std::mutex> lk(g_prof_mu);
    float total = 0.f;
    int n = 0;
    double fl = 0.0, by = 0.0;
    std::vector<ProfRec *> keep;
    for (ProfRec *r : g_prof_recs) {
        if (r->kernel != kernel) { keep.push_back(r); continue; }
        C2M_CUDA(cudaEventSynchronize(r->e1));
        float ms = 0.f;
        C2M_CUDA(cudaEventElapsedTime(&ms, r->e0, r->e1));
        total += ms; fl += r->flops; by += r->bytes; ++n;
        cudaEventDestroy(r->e0);
        cudaEventDestroy(r->e1);
        delete r;
    }
    g_prof_recs.swap(keep);
    *ms_total = total; *launches = n; *flops = fl; *bytes = by;
    return C2M_OK;
}
