// Internal interfaces between the correlation kernels (prep -> search -> rescore).
//
// Data layout in HBM (per feature map of one call, all images b of the batch):
//   p32   [B][HW][Cp]        fp32, pixel-major ("NHWC"), Cp = C rounded up to 8, pad = 0.
//                            Exact values the search is defined on (optionally L2-normalised).
//   hi,lo [B][Cp/8][HW][8]   fp16 split operands of x * 2^sexp[b] (one exponent per map and image):  hi = rn(x*S),
//                            lo = rn(x*S - hi); a non-finite element is written as 0 (its pixel is flagged by ss).
//                            One 16-byte element per (channel-octet, pixel): a (W*8)-wide row of
//                            one image row is contiguous, so a TMA box of (cols*8, rows, octets)
//                            lands in shared memory as [octet][pixel][8 halfs] = the wgmma
//                            K-major no-swizzle core-matrix layout with rows 16 B apart.
//   ss    [B][HW]            fp32 per-pixel sum of squares of p32 * 2^sexp[b]: non-finite iff the pixel holds a
//                            non-finite element (the scaled finite elements are <= 1024, their squares cannot overflow).
//   rinv  [B][NR]            fp32 Ref column scale in SEARCH UNITS (see below): 1 / (||P_r|| 2^sexp_ref + 1e-5 2^sexp_ref)
//                            when is_norm, 1 otherwise; NaN for a Ref patch holding a non-finite element (those are
//                            listed in flag_ref and scored exactly for every query by the rescoring).
//   Search units: both searches score s~ * 2^u, u = sexp_in[b] (+ sexp_ref[b] for raw scores), from the scaled operands,
//   so no product of scales can leave the fp32 range.  u is constant per query, so the ranking is that of s~; the
//   rescoring window is formed in the same units from the scaled norms.
//   part  [B][nchunk][NQ]    Candidate: approximate top-8 (tensor cores) / top-4 (FFMA) of each query over one Ref chunk (nchunk <= 32).
//   ovf   [B*NQ]             (query, chunk bit mask) of the (query, chunk) pairs whose top-2 list may be incomplete:
//                            the exhaustive pass re-scans those chunks exactly (see corr_aux.cu).  Filled from the
//                            front (subject to the re-scan budget) and, for queries whose patch holds a non-finite
//                            element (every chunk, always re-scanned), from the back.
#pragma once
#include "c2m_common.cuh"

namespace c2m {

constexpr int CORR_TOPK = 8;      // candidate slots per (query, Ref chunk): the tensor-core search fills all of them (its window is
                                  // 2^-10-wide because the Ref operand is a plain fp16 rounding), the FFMA search GEN_TOPK
constexpr int GEN_TOPK = 4;
struct __align__(16) Candidate {
    float v[CORR_TOPK];           // approximate scores, best first
    int i[CORR_TOPK];             // Ref patch indices (-1 = empty slot)
    float dropped;                // largest approximate score of the chunk that is NOT in the list
    float pad[3];
};

struct CorrGeom {
    int B, C, Cp;
    int h, w, hr, wr;        // map sizes
    int patch, s_in, s_ref;
    int gh, gw, rh, rw;      // patch grids: input (gh x gw), Ref (rh x rw)
    int NQ, NR;
};

constexpr int CORR_MAX_CHUNKS = 32;

// how a chunk index maps to Ref patches (for the exhaustive fallback)
struct CorrChunkGeom {
    int mode;                // 0: contiguous Ref index ranges of `per` patches (generic search); 1: runs of `per` tiles
    int per;
    int n_rt, rt_x, tile_rows, tile_cols;    // mode 1: tile grid over the Ref patch grid
};

struct CorrOverflow {
    int query;               // b * NQ + q
    unsigned chunks;         // bit c: chunk c must be re-scanned
};

struct CorrWorkspace {
    float *p32_in, *p32_ref;
    __half *hi_in, *lo_in, *hi_ref, *lo_ref;
    float *ss_in, *ss_ref;
    float *rinv;
    Candidate *part;
    CorrOverflow *ovf;       // [B*NQ] overflow list
    unsigned long long *best;   // [B*NQ] packed (exact score, index) of the best candidate so far (best_key)
    float *qnorm;            // [B*NQ] ||P_query|| (exact, deterministic)
    float *qnorm_s;          // [B*NQ] ||P_query|| 2^sexp_in (the window's query scale in search units)
    int *flag_ref;           // [B][NR] Ref patches holding a non-finite element (the first flag_count[b] entries)
    // control block, zeroed at the start of every call (ctl .. ctl + ctl_bytes):
    unsigned *amax_bits;     // [2][B] largest finite |x| per (map, image) (float bits)
    int *sexp;               // [2][B] scale exponents per (map, image): in, ref
    unsigned *ovf_count;     // [2] entries in ovf: [0] from the front, [1] from the back
    unsigned *pr_max_bits;   // [B] max over finite Ref patches of ||P_ref|| 2^sexp_ref rinv (float bits): the window's Ref factor
    unsigned *rinv_max_bits; // [B] max of rinv over finite Ref patches with nonzero norm (float bits)
    unsigned *flag_count;    // [B] entries in flag_ref
    size_t ctl_bytes;
    int nchunk;
    size_t total_bytes;
};

// Sorted top-K insert with a record of what falls off the list: `dropped` ends up as the largest score the chunk
// produced that is not in v[] (scores that never made it, and entries pushed out).  Strict '>' — ties beyond the
// list count as dropped, and the rescoring pass re-scans a chunk exhaustively whenever `dropped` reaches the
// window, so neither ties nor the list length can lose the true argmax.
template <int K>
__device__ __forceinline__ void cand_push(float s, int r, float (&v)[K], int (&i)[K], float &dropped) {
    if (!(s > v[K - 1])) {
        dropped = fmaxf(dropped, s);
        return;
    }
    dropped = fmaxf(dropped, v[K - 1]);
    v[K - 1] = s;
    i[K - 1] = r;
#pragma unroll
    for (int k = K - 1; k > 0; --k) {           // bubble up past strictly smaller entries (stable: ties stay behind)
        const bool up = v[k] > v[k - 1];
        const float tv = v[k - 1];
        const int ti = i[k - 1];
        v[k - 1] = up ? v[k] : tv;
        i[k - 1] = up ? i[k] : ti;
        v[k] = up ? tv : v[k];
        i[k] = up ? ti : i[k];
    }
}
template <int K>
__device__ __forceinline__ void cand_init(float (&v)[K], int (&i)[K]) {
#pragma unroll
    for (int k = 0; k < K; ++k) { v[k] = -INFINITY; i[k] = 0x7fffffff; }
}
template <int K>
__device__ __forceinline__ Candidate cand_pack(const float (&v)[K], const int (&i)[K], float dropped) {
    Candidate c;
#pragma unroll
    for (int k = 0; k < CORR_TOPK; ++k) {
        c.v[k] = k < K ? v[k < K ? k : 0] : -INFINITY;
        c.i[k] = k < K ? (i[k < K ? k : 0] == 0x7fffffff ? -1 : i[k < K ? k : 0]) : -1;
    }
    c.dropped = dropped;
    c.pad[0] = c.pad[1] = c.pad[2] = 0.f;
    return c;
}
// exact scores, torch's max rule: NaN is the maximum, then larger; the lower index wins ties (and among NaNs)
__device__ __forceinline__ bool cand_better(float s, int r, float v, int i) {
    if (s != s) return v == v || r < i;
    return s > v || (s == v && r < i);          // v NaN: both false
}

// (score, index) packed so that an unsigned 64-bit max is cand_better: NaN (one key, whatever its sign and payload)
// above everything, then larger score (-0 as +0), then LOWER index
__device__ __forceinline__ unsigned long long best_key(float s, int r) {
    const unsigned b = __float_as_uint(s == 0.f ? 0.f : s);
    const unsigned ord = s != s ? 0xffffffffu : (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((unsigned long long)ord << 32) | (unsigned long long)(0xffffffffu - (unsigned)r);
}
__device__ __forceinline__ void best_unkey(unsigned long long k, float &s, int &r) {
    const unsigned ord = (unsigned)(k >> 32);
    s = __uint_as_float((ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord);
    r = (int)(0xffffffffu - (unsigned)(k & 0xffffffffu));
}

int corr_prep_launch(const float *x, int B, int C, int Cp, int HW, int l2norm, int map_slot,
                     const CorrWorkspace &ws, float *p32, __half *hi, __half *lo, float *ss,
                     cudaStream_t st);
int corr_rinv_launch(const CorrGeom &g, const CorrWorkspace &ws, int is_norm, cudaStream_t st);
int corr_search_generic_launch(const CorrGeom &g, const CorrWorkspace &ws, cudaStream_t st);
int corr_search_umma_launch(const CorrGeom &g, const CorrWorkspace &ws, cudaStream_t st);
bool corr_umma_supported(const CorrGeom &g);
int corr_umma_pick_nchunk(const CorrGeom &g, int sms);
void corr_umma_chunk_geom(const CorrGeom &g, int nchunk, CorrChunkGeom &cg);
void corr_generic_chunk_geom(const CorrGeom &g, int nchunk, CorrChunkGeom &cg);
// window_coef: rigorous bound on 2 x |approximate - exact score| per unit of ||P_query|| (search units, see corr_aux.cu);
// sub_coef: the same for the absolute rounding of fp16-subnormal operand elements (0 for the fp32 search, see c_abi.cu)
int corr_rescore_launch(const CorrGeom &g, const CorrWorkspace &ws, const CorrChunkGeom &cg, float window_coef,
                        float sub_coef, int is_norm, int norm_input, int64_t *idx, float *val, cudaStream_t st);

}  // namespace c2m
