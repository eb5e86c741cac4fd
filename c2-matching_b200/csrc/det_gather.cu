// Sort and segment steps of the ordered input-gradient gathers (det_gather.cuh).
#include <cub/device/device_radix_sort.cuh>

#include "det_gather.cuh"

namespace c2m {

static int key_bits(long long nkeys) {
    int b = 1;
    while (b < 32 && (1ll << b) < nkeys) ++b;
    return b;
}

static cudaError_t sort_temp_bytes(long long n, long long nkeys, size_t &bytes) {
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
    bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, bytes, k, v, (uint32_t)n, 0, key_bits(nkeys));
}

cudaError_t det_layout(void *base, long long n, long long nkeys, DetLayout &L) {
    size_t off = 0;
    unsigned char *p = static_cast<unsigned char *>(base);
    auto take = [&](size_t bytes) {
        void *r = p ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    for (int i = 0; i < 2; ++i) L.keys[i] = static_cast<uint32_t *>(take((size_t)n * 4));
    for (int i = 0; i < 2; ++i) L.vals[i] = static_cast<uint32_t *>(take((size_t)n * 4));
    L.seg = static_cast<uint32_t *>(take((size_t)nkeys * 4));
    const cudaError_t e = sort_temp_bytes(n, nkeys, L.temp_bytes);
    L.temp = take(L.temp_bytes);
    L.total = off;
    return e;
}

// seg[key] = number of sorted keys below `key` (lower bound)
__global__ void det_segments_kernel(const uint32_t *__restrict__ keys, uint32_t n, uint32_t nkeys,
                                    uint32_t *__restrict__ seg) {
    for (uint32_t key = blockIdx.x * blockDim.x + threadIdx.x; key < nkeys; key += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (keys[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        seg[key] = lo;
    }
}

int det_sort_segments(DetLayout &L, uint32_t n, uint32_t nkeys, int &sorted, cudaStream_t st) {
    size_t need = 0;
    C2M_CUDA(sort_temp_bytes(n, nkeys, need));
    C2M_CHECK_ARG(need <= L.temp_bytes, "ordered gather: sort needs %zu temporary bytes, %zu reserved", need,
                  L.temp_bytes);
    cub::DoubleBuffer<uint32_t> k(L.keys[0], L.keys[1]), v(L.vals[0], L.vals[1]);
    size_t temp_bytes = L.temp_bytes;
    C2M_CUDA(cub::DeviceRadixSort::SortPairs(L.temp, temp_bytes, k, v, n, 0, key_bits(nkeys), st));
    C2M_LAUNCH_CHECK("cub::DeviceRadixSort::SortPairs");
    sorted = k.selector;
    det_segments_kernel<<<grid_blocks(nkeys), 256, 0, st>>>(k.Current(), n, nkeys, L.seg);
    C2M_LAUNCH_CHECK("det_segments_kernel");
    return C2M_OK;
}

static bool pass_fits_32bit(long long planes, long long entries_per_plane, long long keys_per_plane) {
    return planes * entries_per_plane <= 0xFFFFFFFFll && planes * keys_per_plane <= 0xFFFFFFFFll;
}

bool det_plane_fits(long long entries, long long keys, const char *who) {
    if (pass_fits_32bit(1, entries, keys)) return true;
    set_error("%s: a plane of %lld entries exceeds the 32-bit entry id", who, entries);
    return false;
}

size_t det_workspace_bytes(long long planes, long long nplanes, long long entries_per_plane, long long keys_per_plane,
                           const char *who) {
    if (planes > nplanes) planes = nplanes;
    if (planes < 1) planes = 1;
    if (!pass_fits_32bit(planes, entries_per_plane, keys_per_plane)) {
        set_error("%s: %lld planes of %lld entries and %lld pixels exceed the 32-bit entry id", who, planes,
                  entries_per_plane, keys_per_plane);
        return 0;
    }
    DetLayout L;
    const cudaError_t e = det_layout(nullptr, planes * entries_per_plane, planes * keys_per_plane, L);
    if (e != cudaSuccess) {
        set_error("%s: sort workspace query failed: %s", who, cudaGetErrorString(e));
        return 0;
    }
    return L.total;
}

int det_planes_per_pass(size_t ws_bytes, long long nplanes, long long entries_per_plane, long long keys_per_plane) {
    long long lo = 0, hi = nplanes;         // lo fits (0 trivially), find the largest that does
    while (lo < hi) {
        const long long mid = lo + (hi - lo + 1) / 2;
        DetLayout L;
        const bool fits = pass_fits_32bit(mid, entries_per_plane, keys_per_plane) &&
                          det_layout(nullptr, mid * entries_per_plane, mid * keys_per_plane, L) == cudaSuccess &&
                          L.total <= ws_bytes;
        if (fits) lo = mid;
        else hi = mid - 1;
    }
    return (int)lo;
}

}  // namespace c2m
