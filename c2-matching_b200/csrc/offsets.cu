// idx -> 9-shift pre-offset pyramid for one scale (a4 + a5 of SURVEY.md §8).
//
// Replaces CorrespondenceGenerationArch.index_to_flow + the tensor_shift / repeat_interleave
// cascade (mmsr/models/archs/corres_generation_arch.py:29-46,70-104; arch_util.py:291-315): ~40
// tiny elementwise kernels and a meshgrid per image become one launch per scale for the batch.  The
// decode itself is pyramid_flow (dcn_sampling.cuh), which the fused DCN forward also calls.
#include "dcn_sampling.cuh"

namespace c2m {

__global__ void offset_pyramid_kernel(const long long *__restrict__ idx, int gh, int gw, int ref_gw, int s,
                                      float2 *__restrict__ out) {
    const int HS = (gh + 2) * s, WS = (gw + 2) * s;
    const int b = blockIdx.z, k = blockIdx.y;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < HS * WS; e += gridDim.x * blockDim.x)
        out[((long long)b * 9 + k) * HS * WS + e] = pyramid_flow(idx, b, gh, gw, ref_gw, s, e / WS, e % WS, k / 3, k % 3);
}

}  // namespace c2m

extern "C" int c2m_offset_pyramid_f32(const int64_t *idx, int B, int gh, int gw, int ref_gw, int scale, float *out,
                                      c2m_stream_t stream) {
    C2M_CHECK_ARG(idx && out, "offset_pyramid: null pointer");
    C2M_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && ref_gw > 0 && scale > 0, "offset_pyramid: bad shape");
    const int n = (gh + 2) * scale * (gw + 2) * scale;
    int bx = c2m::ceil_div(n, 256);
    if (bx > 1024) bx = 1024;
    dim3 grid(bx, 9, B);
    c2m::offset_pyramid_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(idx), gh, gw, ref_gw, scale, reinterpret_cast<float2 *>(out));
    C2M_LAUNCH_CHECK("offset_pyramid_kernel");
    return C2M_OK;
}
