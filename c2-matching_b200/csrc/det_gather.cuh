// Shared machinery of the ordered input-gradient gathers (dcn_bwd.cu, psroi.cu), used when torch's deterministic
// algorithms are enabled in place of the atomicAdd scatters.
//
// Each contribution to an input plane is an entry with a 32-bit id that encodes its place in the summation order.
// A pass over `np` planes:
//   1. the op's emit kernel writes one (key, id) pair per entry, entries of plane q at [q * E, (q + 1) * E) in
//      ascending id, key = q * (HW + 1) + pixel, or q * (HW + 1) + HW ("no pixel") for an entry that contributes
//      nothing;
//   2. a stable radix sort by key (cub::DeviceRadixSort, stable) leaves every pixel's ids ascending;
//   3. seg[key] = first sorted position with a key >= key, for key in [0, np * (HW + 1));
//   4. the op's gather kernel walks seg[key] .. seg[key + 1] of each pixel and adds in that order.
// The caller-owned workspace holds the four pair arrays, seg and CUB's temporary storage; planes per pass are as many
// as it holds (at least one).
#pragma once
#include "c2m_common.cuh"

namespace c2m {

struct DetLayout {
    uint32_t *keys[2], *vals[2], *seg;
    void *temp;
    size_t temp_bytes, total;
};

// Workspace layout of a pass of n entries and nkeys keys; base may be null (size query).  CUB's size query reads the
// current device.
cudaError_t det_layout(void *base, long long n, long long nkeys, DetLayout &L);

// Steps 2 and 3 on the arrays of L: sorts L.keys[0] / L.vals[0] (n pairs) and fills L.seg.  On return `sorted` is the
// index (0 or 1) of the buffers that hold the sorted pairs.
int det_sort_segments(DetLayout &L, uint32_t n, uint32_t nkeys, int &sorted, cudaStream_t st);

// Largest planes-per-pass in [1, nplanes] whose layout fits ws_bytes (entries_per_plane / keys_per_plane each), or 0
// when even one plane does not fit.
int det_planes_per_pass(size_t ws_bytes, long long nplanes, long long entries_per_plane, long long keys_per_plane);

// Bytes for `planes` planes per pass (clamped to [1, nplanes]); 0 with the error set when a pass exceeds the 32-bit
// entry or key range.
size_t det_workspace_bytes(long long planes, long long nplanes, long long entries_per_plane, long long keys_per_plane,
                           const char *who);

// False, with the error set, when one plane of `entries` entries and `keys` keys exceeds the 32-bit entry id.
bool det_plane_fits(long long entries, long long keys, const char *who);

// Steps 1-4 over `nplanes` planes of E entries and K keys each, as many planes per pass as ws_bytes holds:
// emit(q0, n, keys, ids) writes the pairs of planes [q0, q0 + n), gather(q0, n, seg, ids) adds them up from the
// segment starts and the sorted ids.  Both return a status.
template <typename Emit, typename Gather>
int det_passes(void *ws, size_t ws_bytes, long long nplanes, long long E, long long K, const char *who,
               cudaStream_t st, Emit emit, Gather gather) {
    C2M_CHECK_ARG(ws, "%s: null workspace", who);
    const int np = det_planes_per_pass(ws_bytes, nplanes, E, K);
    C2M_CHECK_ARG(np >= 1, "%s: workspace of %zu bytes holds no plane (%zu needed)", who, ws_bytes,
                  det_workspace_bytes(1, nplanes, E, K, who));
    DetLayout L;
    C2M_CUDA(det_layout(ws, np * E, np * K, L));
    for (long long q0 = 0; q0 < nplanes; q0 += np) {
        const int n = (int)(nplanes - q0 < np ? nplanes - q0 : np);
        if (int rc = emit((int)q0, n, L.keys[0], L.vals[0])) return rc;
        int sorted;
        if (int rc = det_sort_segments(L, (uint32_t)(n * E), (uint32_t)(n * K), sorted, st)) return rc;
        if (int rc = gather((int)q0, n, L.seg, L.vals[sorted])) return rc;
    }
    return C2M_OK;
}

}  // namespace c2m
