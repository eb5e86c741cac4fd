/*
 * libc2m_sm100 — C ABI of the H100-native C2-Matching restoration-forward hot path.
 *
 * Plain C: raw device pointers, sizes, a CUDA stream handle, int status.  No torch / ATen
 * types.  Every entry point is asynchronous on `stream`, re-entrant (no global scratch: the
 * caller owns outputs and the workspace) and takes the device from the current CUDA context,
 * which is what the reference's operator boundary assumes (it launches on the current stream
 * of the tensors' device under the GIL, DCNv2/src/cuda/dcn_v2_cuda.cu:107,139).
 *
 * Reference interfaces replaced (paths relative to the reference repo root):
 *   c2m_deform_conv_{forward,im2col,col2im_coord,col2im,col2im_det}_{f32,f64}
 *                                   <- `_ext.dcn_v2_forward` / `_ext.dcn_v2_backward`
 *                                      mmsr/models/archs/DCNv2/src/vision.cpp:3-8 (pybind export),
 *                                      src/dcn_v2.h:9-72 (dispatch), src/cuda/dcn_v2_cuda.cu:42-335;
 *                                      and `deform_conv_cuda` (DCNv1 and grouped DCNv2)
 *                                      mmsr/models/archs/dcn/src/deform_conv_cuda.cpp:151-695,
 *                                      src/deform_conv_cuda_kernel.cu
 *   c2m_dcn_v2_fused_forward_f32    <- DCN_sep_pre_multi_offset.forward (everything after the
 *                                      conv_offset_mask conv) mmsr/models/archs/DCNv2/dcn_v2.py:229-253
 *   c2m_corr_argmax_f32             <- feature_match_index  mmsr/models/archs/ref_map_util.py:26-86
 *                                      (+ optional fused per-pixel channel L2 normalisation,
 *                                      mmsr/models/archs/corres_generation_arch.py:56-58)
 *   c2m_offset_pyramid_f32          <- index_to_flow + 9-shift x scale pyramid
 *                                      mmsr/models/archs/corres_generation_arch.py:29-46,70-104
 *   c2m_psroi_pooling_{forward,backward}_{f32,f64}
 *                                   <- `_ext.dcn_v2_psroi_pooling_forward` / `_backward`
 *                                      src/dcn_v2.h:75-144, src/cuda/dcn_v2_psroi_pooling_cuda.cu:58-419
 *
 * The Python binding a reference maintainer would add is shown in INTEGRATION.md.
 */
#ifndef C2M_SM100_H
#define C2M_SM100_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* same object as cudaStream_t / CUstream */
typedef struct CUstream_st *c2m_stream_t;

/* status codes (0 = ok).  c2m_last_error() returns a thread-local description. */
enum {
    C2M_OK = 0,
    C2M_ERR_INVALID = 1,      /* bad shape / argument (reference: AT_ASSERTM -> RuntimeError) */
    C2M_ERR_WORKSPACE = 2,    /* workspace missing or too small */
    C2M_ERR_CUDA = 3,         /* CUDA runtime / launch failure (reference only printf'd these) */
    C2M_ERR_UNSUPPORTED = 4   /* no sm_90 device / driver entry point missing */
};

int c2m_abi_version(void);      /* 7 since grad_output takes one exponent per image: gy_amax holds [B] values,
                                 * c2m_grad_psa_from_f32 and c2m_grad_unscale_f32 are gone (6: the fp32 c2m_dcn_v2_*
                                 * twins of c2m_deform_conv_* are gone; 5: c2m_dcn_tc_args
                                 * takes only x_il; 4: .x_il / c2m_psa_interleave; 3: .mask; 2: out_f32_octets /
                                 * om_octets).  Later additions (c2m_dcn_tc_args.x_amax / .mask_amax,
                                 * c2m_dcn_tc_operand_*, c2m_conv3x3_args.x_amax with c2m_conv3x3_operand_f32 and
                                 * c2m_conv3x3_wgrad_scaled) come with new symbols that an older library lacks. */
const char *c2m_last_error(void);

/* --- correlation / index_map --------------------------------------------------------------
 * For b in [0,B):  idx[b,q] = argmax_r < P_in(b,q), P_ref(b,r) / (||P_ref(b,r)|| + 1e-5) >
 * over the Ref patch grid (lowest r on ties), val[b,q] = that maximum (divided by
 * ||P_in(b,q)|| + 1e-5 when norm_input).  fin [B,C,h,w], fref [B,C,hr,wr] fp32 NCHW;
 * idx int64 [B,h',w'], val fp32 [B,h',w'], h' = (h-patch)/s_in+1.  B = 1 is the reference call.
 *
 * l2norm != 0 first applies x[:,p] / max(||x[:,p]||, 1e-12) to both maps (the caller's
 * F.normalize in the reference).
 *
 * flags: bit0 = force the generic CUDA-core search instead of the tensor-core kernel.
 * The tensor-core search proposes candidates; the returned idx/val always come from the exact
 * (double-accumulated, float-rounded) rescoring pass, so they do not depend on tensor-core
 * rounding.
 */
size_t c2m_corr_workspace_bytes(int B, int C, int h, int w, int hr, int wr, int patch, int s_in, int s_ref);

int c2m_corr_argmax_f32(const float *fin, const float *fref, int B, int C, int h, int w, int hr, int wr,
                        int patch, int s_in, int s_ref, int is_norm, int norm_input, int l2norm,
                        unsigned flags, int64_t *idx, float *val, void *ws, size_t ws_bytes,
                        c2m_stream_t stream);

/* --- idx -> pre-offset pyramid ------------------------------------------------------------
 * idx [B,gh,gw] -> out [B,9,s*(gh+2),s*(gw+2),2] fp32, last dim (x,y);  tap k=3i+j is the flow
 * map scaled by s, nearest-upsampled by s and shifted down/right by (s*i, s*j), zero filled.
 * ref_gw: patch-grid width used to decode idx (the reference uses gw, the INPUT grid width).
 */
int c2m_offset_pyramid_f32(const int64_t *idx, int B, int gh, int gw, int ref_gw, int scale, float *out,
                           c2m_stream_t stream);

/* --- deformable convolution on the CUDA cores, v1 and modulated, with conv groups -------------------------------
 * (`_ext.dcn_v2_forward` / `_backward` call the fp32 entries with groups = 1 and a mask; `deform_conv_cuda`,
 * mmsr/models/archs/dcn/src, calls all of them.)
 * out[b,o,p] = bias[o] + sum_{c,i,j} W[o,c',i,j] * mask[b,g(c)*kh*kw+i*kw+j,p] *
 *              bilinear(x[b,c], ho*sh-ph+i*dh+off_y, wo*sw-pw+j*dw+off_x)
 * over the input channels c of o's conv group, c' = c - (first channel of that group);
 * off_y/off_x = offset[b, 2*(g(c)*kh*kw+i*kw+j) (+1), p];  sample is 0 unless
 * -1 < y < H and -1 < x < W; g(c) = c / (C/dg).
 *   groups: weight [Cout, C/groups, kh, kw]; output channel o reads the input channels of its conv group
 *           o / (Cout/groups).  Conv groups and deformable groups partition C independently.
 *   mask == NULL: modulation 1 (DCNv1); then grad_mask must be NULL too.  bias == NULL adds nothing.
 * Every tensor of one call is fp32 (_f32) or fp64 (_f64); positions are computed in the dtype, like the reference's
 * `scalar_t` kernels.
 * Forward: x [B,C,H,W]; element (b,c,y,x) at x[b*xs_b + c*xs_c + y*xs_y + x*xs_x] (element strides, so
 * NCHW-contiguous and channels-last storage are both accepted); out [B,Cout,Ho,Wo]: element strides os_b, os_c,
 * os_y, os_x likewise.  offset [B,2*dg*kh*kw,Ho,Wo], mask [B,dg*kh*kw,Ho,Wo], weight, bias [Cout]: contiguous.
 * Backward pieces: every tensor NCHW-contiguous; shape->x* / o* strides are ignored.  The two dense GEMMs are the
 * caller's, per conv group:
 *   columns [B, C*kh*kw, Ho*Wo] = mask * bilinear(x)                      (for grad_weight = gout x columns^T)
 *   gcol    [B, C*kh*kw, Ho*Wo] = W^T x grad_output                       (computed by the caller)
 *   grad_offset [B,2*dg*kh*kw,Ho,Wo], grad_mask [B,dg*kh*kw,Ho,Wo] written; grad_input [B,C,H,W] ACCUMULATED
 *   (caller zero-fills it first), or written in a fixed order by c2m_deform_conv_col2im_det_* (see "ordered input
 *   gradients" below).
 * Rejected with C2M_ERR_INVALID: empty tensors or output, kernel sizes / strides / dilations < 1, C not divisible by
 * dg, groups < 1, C or Cout not divisible by groups.
 */
typedef struct {
    int B, C, H, W, Cout;
    int kh, kw, sh, sw, ph, pw, dh, dw, dg;
    long long xs_b, xs_c, xs_y, xs_x;
    long long os_b, os_c, os_y, os_x;
} c2m_dcn_shape;

int c2m_deform_conv_forward_f32(const float *x, const float *offset, const float *mask, const float *weight,
                                const float *bias, int groups, float *out, const c2m_dcn_shape *shape,
                                c2m_stream_t stream);
int c2m_deform_conv_forward_f64(const double *x, const double *offset, const double *mask, const double *weight,
                                const double *bias, int groups, double *out, const c2m_dcn_shape *shape,
                                c2m_stream_t stream);
int c2m_deform_conv_im2col_f32(const float *x, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                               float *columns, c2m_stream_t stream);
int c2m_deform_conv_im2col_f64(const double *x, const double *offset, const double *mask, const c2m_dcn_shape *shape,
                               double *columns, c2m_stream_t stream);
int c2m_deform_conv_col2im_coord_f32(const float *gcol, const float *x, const float *offset, const float *mask,
                                     const c2m_dcn_shape *shape, float *grad_offset, float *grad_mask,
                                     c2m_stream_t stream);
int c2m_deform_conv_col2im_coord_f64(const double *gcol, const double *x, const double *offset, const double *mask,
                                     const c2m_dcn_shape *shape, double *grad_offset, double *grad_mask,
                                     c2m_stream_t stream);
int c2m_deform_conv_col2im_f32(const float *gcol, const float *offset, const float *mask, const c2m_dcn_shape *shape,
                               float *grad_input, c2m_stream_t stream);
int c2m_deform_conv_col2im_f64(const double *gcol, const double *offset, const double *mask,
                               const c2m_dcn_shape *shape, double *grad_input, c2m_stream_t stream);

/* Fused DCN_sep_pre_multi_offset tail, the forward above in fp32 with groups = 1, where
 * `om` = conv_offset_mask(feat) [B,3*dg*kh*kw,Ho,Wo] raw;
 *   off_y = om[2j] + pre[...,1], off_x = om[2j+1] + pre[...,0], mask = sigmoid(om[2*dg*kh*kw + j]),
 *   j = g*kh*kw + k;  pre = pre_offset [B,kh*kw,Ho,Wo,2] (x,y) or NULL.
 * If pre == NULL and idx != NULL the pre-offsets are rebuilt on the fly from idx [B,gh,gw]
 * (pyramid scale `pre_scale`, decode width ref_gw) exactly as c2m_offset_pyramid_f32 would.
 * lrelu_slope: out = v > 0 ? v : slope*v applied when lrelu_slope != 1 (pass 1.f for none).
 */
int c2m_dcn_v2_fused_forward_f32(const float *x, const float *om, const float *pre, const int64_t *idx,
                                 int gh, int gw, int ref_gw, int pre_scale, const float *weight,
                                 const float *bias, float lrelu_slope, float *out,
                                 const c2m_dcn_shape *shape, c2m_stream_t stream);

/* --- plain 3x3 / stride 1 / pad 1 convolution on the tensor cores (wgmma), fp32-grade (split fp16 x 3) -------
 * (SURVEY.md §8f N3: every plain convolution of RestorationNet / the VGG trunks; the reference
 * runs them through cuDNN, e.g. arch_util.py:80-136, ref_restoration_arch.py:147-187.)
 * Activations travel between these convolutions in the packed-split layout "PSA":
 *     hi, lo : fp16 [B][ceil(C/8)][H][W][8],   value = (hi + lo) * 2^-sa
 * c2m_psa_from_f32 / c2m_psa_to_f32 convert from / to strided fp32 ([B,C,H,W] with element
 * strides; to_f32 can add a strided fp32 tensor of the same strides).
 * Weights [Cout,Cin,3,3] fp32 are packed once (c2m_conv3x3_pack_weights_f32) into a blob of
 * c2m_conv3x3_packed_weight_bytes(Cin,Cout) bytes (Cin = total input channels).
 *     y = act(conv(cat[in, in2], W) + bias)          act: 0 none, 1 ReLU, 2 LeakyReLU(0.1)
 *     PSA output  (optional): y + res + res2, or PixelShuffle(2)(y) when pixel_shuffle == 2
 *     fp32 output (optional): y + add_f32, strided [B,Cout,H,W]; or, with out_f32_octets != 0, y in the
 *     octet-planar fp32 layout [B][ceil(Cout/8)][H][W][8] (strides and add_f32 unused; padding channels 0)
 *     that c2m_dcn_v2_fused_tc reads its `om` operand from (om_octets)
 * Any Cin / Cout; in2 (optional) is concatenated after in along channels (then Cin % 32 == 0).
 * Needs H >= 18 and W >= 10.
 */
typedef struct {
    const void *in_hi, *in_lo;   int Cin;
    const void *in2_hi, *in2_lo; int Cin2;
    int B, H, W, sa_in;
    const void *packed_w; const float *bias; int Cout; int act;
    const void *res_hi, *res_lo, *res2_hi, *res2_lo; int sa_res;
    void *out_hi, *out_lo; int sa_out; int pixel_shuffle;
    float *out_f32; const float *add_f32; long long os_b, os_c, os_y, os_x;
    int out_f32_octets;
    const unsigned *x_amax;     /* [B] or NULL (then sa_in applies): per-image input exponents, the amax written by
                                 * c2m_conv3x3_operand_f32 together with in_hi / in_lo; the epilogue divides image b by
                                 * 2^(14 - floor(log2 x_amax[b])) (0 for an all-zero image).  One input only. */
} c2m_conv3x3_args;

size_t c2m_conv3x3_packed_weight_bytes(int Cin, int Cout);
int c2m_conv3x3_pack_weights_f32(const float *w, int Cin, int Cout, void *packed, c2m_stream_t stream);
int c2m_psa_from_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c, long long xs_y,
                     long long xs_x, int sa, void *hi, void *lo, c2m_stream_t stream);
int c2m_psa_to_f32(const void *hi, const void *lo, int B, int C, int H, int W, int sa, const float *add, float *out,
                   long long os_b, long long os_c, long long os_y, long long os_x, c2m_stream_t stream);
int c2m_conv3x3(const c2m_conv3x3_args *args, c2m_stream_t stream);
/* Operand of the differentiable convolution, for x and for grad_output: x [B,C,H,W] fp32 (element strides) of any magnitude -> PSA hi / lo holding
 * image b times 2^sa_b, sa_b = 14 - floor(log2 amax[b]), where amax[b], the largest finite |x| of image b (NaN and Inf
 * do not count; 0 gives sa_b = 0; sa_b is clamped to +-120), is computed on the device and its fp32 bits stored in
 * amax[0, B) (device memory).  Pass amax as c2m_conv3x3_args.x_amax and to c2m_conv3x3_wgrad_scaled.  Scaling an image by
 * 2^k leaves its PSA planes bit for bit the same, so the output and the gradients scale by exactly 2^k while in range. */
int c2m_conv3x3_operand_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c, long long xs_y,
                            long long xs_x, void *hi, void *lo, unsigned *amax, c2m_stream_t stream);
/* Backward of the convolution above (3x3 / stride 1 / pad 1, one input), fp32-grade, no host synchronisation.
 * grad_output g [B,C,H,W] enters as c2m_conv3x3_operand_f32(g, ..., hi, lo, gy_amax): one exponent per image, so an
 * image's gradients do not depend on the other images' magnitudes.
 * Input gradient: c2m_conv3x3 of that PSA tensor with x_amax = gy_amax (Cin = the forward's Cout, Cout = the forward's
 *   Cin) and the weights W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx] packed by c2m_conv3x3_pack_weights_f32, fp32 output.
 * c2m_conv3x3_wgrad: dW[co][ci][ky][kx] = sum over b, y, x of g[b,co,y,x] * x[b,ci,y+ky-1,x+kx-1] (zero outside the
 *   map), written to dw [Cout,Cin,3,3] fp32.  gy_* / gy_amax ([B]): the output of c2m_conv3x3_operand_f32; x_*: the forward's
 *   input as PSA at scale exponent 0 (c2m_conv3x3_wgrad) or, with x_amax, the output of c2m_conv3x3_operand_f32
 *   (c2m_conv3x3_wgrad_scaled).  Only pixels inside the map contribute, also next to a non-finite x.  Split-K over CTAs with per-CTA partials in `ws` (at least
 *   c2m_conv3x3_wgrad_workspace_bytes(B, Cin, Cout, H, W) bytes, which depends on the device's SM count), summed in one
 *   fixed order: the same bits on every run on a given device.  Needs H >= 18 and W >= 10, like c2m_conv3x3.
 */
size_t c2m_conv3x3_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W);   /* 0 on a bad shape */
int c2m_conv3x3_wgrad(const void *gy_hi, const void *gy_lo, const unsigned *gy_amax, const void *x_hi, const void *x_lo,
                      int B, int Cin, int Cout, int H, int W, float *dw, void *ws, size_t ws_bytes,
                      c2m_stream_t stream);
int c2m_conv3x3_wgrad_scaled(const void *gy_hi, const void *gy_lo, const unsigned *gy_amax, const void *x_hi,
                             const void *x_lo, const unsigned *x_amax, int B, int Cin, int Cout, int H, int W,
                             float *dw, void *ws, size_t ws_bytes, c2m_stream_t stream);
/* MaxPool2d(2, 2) on a PSA tensor (floor semantics: odd trailing row / column dropped), PSA result. */
int c2m_psa_maxpool2(const void *hi, const void *lo, int B, int C, int H, int W, void *out_hi, void *out_lo,
                     c2m_stream_t stream);

/* --- DCNv2 forward on the tensor cores (wgmma) (3x3 / stride 1 / pad 1 / dilation 1, C/dg % 8 == 0, Cout <= 256) ---
 * Same contract as c2m_dcn_v2_fused_forward_f32 (raw conv_offset_mask output `om`, pre-offsets from
 * `pre` or rebuilt from `idx`), but the contraction runs as a split-fp16 tensor-core GEMM fed by
 * gather warps; the input `x_il` is a PSA tensor (see c2m_psa_from_f32) with the two halves of a (pixel, octet)
 * adjacent, fp16 [B][C/8][H][W][hi 8 | lo 8] (c2m_dcn_tc_operand_psa), 32 B aligned: its octet-planar layout lets a
 * warp's corner fetches share cache lines, and a corner fetch is one 32 B sector.  Outputs: PSA (out_hi/out_lo) and / or
 * strided fp32; `lrelu` != 0 applies LeakyReLU(0.1).  Weights are packed once with
 * c2m_dcn_tc_pack_weights_f32 into c2m_dcn_tc_packed_weight_bytes(C, Cout, dg) bytes.
 * An fp32 input of any magnitude goes through c2m_dcn_tc_operand_f32, which writes x_il as x * 2^sa with a
 * per-image exponent sa (amax * 2^sa in [2^11, 2^12), from the exponent bits of the image's largest finite |x|) and
 * stores the amax bits in amax[0, B) (and, given the final mask, the mask's in amax[B, 2B)); pass x_amax = amax (and
 * mask_amax = amax + B) here: the epilogue divides 2^sa back out image by image, and the gather scales each image's
 * mask to max |mask| in [1, 2).  Computed on the device (no host synchronisation); NULL means exponent 0.
 * x_il holds c2m_dcn_tc_operand_bytes(B, C, H, W, dg) bytes: the operand, then a zero tail that both operand writers
 * fill and that the gather reads for a sample outside the window and a corner outside the image, so those contribute
 * exactly 0 and, as in the reference, the image is not read for them.
 */
typedef struct {
    const void *x_il;
    const float *om; const float *pre; const int64_t *idx;
    int gh, gw, ref_gw, pre_scale;
    int B, C, H, W, Cout, dg;
    const void *packed_w; const float *bias; int lrelu;
    void *out_hi, *out_lo; int sa_out;
    float *out_f32; long long os_b, os_c, os_y, os_x;
    int om_octets;               /* != 0: om is octet-planar fp32 [B][ceil(27*dg/8)][H][W][8] */
    const float *mask;           /* != NULL: the `_ext.dcn_v2_forward` contract (DCNv2/src/dcn_v2.h:9-22) — `om` is the
                                  * FINAL offset tensor [B,2*dg*9,H,W], `mask` the FINAL modulation [B,dg*9,H,W]
                                  * (no sigmoid applied); pre, idx and om_octets must be unset */
    const unsigned *x_amax;      /* [B] or NULL: written by c2m_dcn_tc_operand_f32 together with x_il */
    const unsigned *mask_amax;   /* [B] or NULL (needs mask): written by c2m_dcn_tc_operand_f32 given the mask */
} c2m_dcn_tc_args;

int c2m_dcn_tc_supported(int C, int Cout, int dg);
size_t c2m_dcn_tc_packed_weight_bytes(int C, int Cout, int dg);
int c2m_dcn_tc_pack_weights_f32(const float *w, int C, int Cout, int dg, void *packed, c2m_stream_t stream);
int c2m_dcn_v2_fused_tc(const c2m_dcn_tc_args *args, c2m_stream_t stream);
/* Bytes of x_il for c2m_dcn_v2_fused_tc: B*C*H*W*2 fp16 of operand, then the zero tail (0 if unsupported). */
size_t c2m_dcn_tc_operand_bytes(int B, int C, int H, int W, int dg);
/* PSA hi / lo planes (scale exponent 0) -> x_il: interleaved [B][C/8][H][W][hi 8 | lo 8] and its zero tail. */
int c2m_dcn_tc_operand_psa(const void *hi, const void *lo, int B, int C, int H, int W, int dg, void *x_il,
                           c2m_stream_t stream);
/* fp32 x [B,C,H,W] (element strides; dense NCHW or channels-last) -> x_il (operand * 2^sa and zero tail) and amax[B]
 * (bits of each image's largest finite |x|); with mask != NULL (the final mask [B,dg*9,H,W], contiguous) also
 * amax[B + b] for the mask.  NaN and Inf do not count towards a maximum. */
int c2m_dcn_tc_operand_f32(const float *x, int B, int C, int H, int W, long long xs_b, long long xs_c, long long xs_y,
                           long long xs_x, int dg, const float *mask, void *x_il, unsigned *amax, c2m_stream_t stream);

/* --- Backward of the tensor-core DCN (the `_ext` contract: final offsets and final mask) -------------------------
 * Same shapes as c2m_dcn_v2_fused_tc (c2m_dcn_tc_supported), maps of at least 16 x 8.  Inputs:
 *   gy_hi / gy_lo / gy_amax   grad_output [B,Cout,H,W] as c2m_conv3x3_operand_f32 writes it: PSA image b times
 *                             2^sg_b, gy_amax [B]
 *   x_il, x_amax, mask_amax   the forward's operand: c2m_dcn_tc_operand_f32(x, ..., mask, x_il, amax) with
 *                             x_amax = amax, mask_amax = amax + B
 *   offset, mask              final offsets [B,2*dg*9,H,W] and final mask [B,dg*9,H,W], contiguous fp32
 * c2m_dcn_tc_dgrad computes gcol = W^T gY on the tensor cores without storing it and writes grad_offset (shape of
 * offset) and grad_mask (shape of mask), each element once in a fixed order.  With grad_input != NULL it also ADDS
 * the input gradient into grad_input [B,C,H,W] (contiguous, caller zero-fills) with atomics.  packed_w: the weights
 * packed by c2m_dcn_tc_pack_dgrad_weights_f32 into c2m_dcn_tc_dgrad_packed_weight_bytes(C, Cout, dg) bytes.
 * c2m_dcn_tc_wgrad writes grad_weight [Cout,C,3,3], bitwise reproducible on a given device, using a workspace of
 * c2m_dcn_tc_wgrad_workspace_bytes(B, C, H, W, Cout, dg) bytes (0 on bad arguments; it queries the current device). */
typedef struct {
    const void *gy_hi, *gy_lo;
    const unsigned *gy_amax;     /* [B] */
    const void *x_il;
    const unsigned *x_amax, *mask_amax;
    const float *offset, *mask;
    int B, C, H, W, Cout, dg;
    const void *packed_w;        /* dgrad */
    float *grad_offset, *grad_mask, *grad_input;   /* dgrad; grad_input may be NULL */
    float *grad_weight;          /* wgrad */
    void *ws;                    /* wgrad */
    size_t ws_bytes;
} c2m_dcn_tc_grad_args;

size_t c2m_dcn_tc_dgrad_packed_weight_bytes(int C, int Cout, int dg);
int c2m_dcn_tc_pack_dgrad_weights_f32(const float *w, int C, int Cout, int dg, void *packed, c2m_stream_t stream);
int c2m_dcn_tc_dgrad(const c2m_dcn_tc_grad_args *args, c2m_stream_t stream);
size_t c2m_dcn_tc_wgrad_workspace_bytes(int B, int C, int H, int W, int Cout, int dg);
int c2m_dcn_tc_wgrad(const c2m_dcn_tc_grad_args *args, c2m_stream_t stream);

/* --- ordered input gradients (used when torch's deterministic algorithms are enabled) -----------------------------
 * Same results as the col2im / PS-ROI grad_input scatters above, except that every element of grad_input is a sum in
 * one fixed order, so it is the same bit for bit on every run, and that grad_input is WRITTEN (every element, +0
 * where nothing contributes), not accumulated.  Each contribution is the scatter's own expression; an element starts
 * at +0 and adds its contributions with correctly rounded adds in this order:
 *   DCN (c2m_deform_conv_col2im_det_{f32,f64}; arguments as c2m_deform_conv_col2im_*): over the
 *     sampling points of deformable group c / (C/dg) of image b, ascending tap, then output pixel, then corner
 *     (low-low, low-high, high-low, high-high); in-image corners only.
 *   PS-ROI (c2m_psroi_pooling_grad_input_det_{f32,f64}; arguments as the backward, without input and grad_trans): over
 *     the ROIs with batch index b, ascending ROI, then bin (row-major), then sample (row-major), then corner (floor,
 *     +y, +x, +x+y), skipping dropped samples, corners that coincide with the floor corner and outputs with count <= 0.
 * A plane is one (image, deformable group) for DCN and one (image, class) for PS-ROI.  The workspace is caller-owned:
 * c2m_*_det_workspace_bytes(shape, planes) is the size that processes `planes` planes per pass (clamped to
 * [1, planes in the call]); the entry points process as many planes per pass as ws_bytes holds, at least one.  The
 * one-plane size does not depend on B.  A plane of 2^32 or more contributions is rejected (C2M_ERR_INVALID; the
 * queries return 0).  The size queries ask CUB for its sort storage and so need a current CUDA device. */
size_t c2m_dcn_col2im_det_workspace_bytes(const c2m_dcn_shape *shape, int planes);
int c2m_deform_conv_col2im_det_f32(const float *gcol, const float *offset, const float *mask,
                                   const c2m_dcn_shape *shape, float *grad_input, void *ws, size_t ws_bytes,
                                   c2m_stream_t stream);
int c2m_deform_conv_col2im_det_f64(const double *gcol, const double *offset, const double *mask,
                                   const c2m_dcn_shape *shape, double *grad_input, void *ws, size_t ws_bytes,
                                   c2m_stream_t stream);

/* --- deformable PS-ROI pooling (`_ext.dcn_v2_psroi_pooling_forward` / `_backward`) -------------------------------
 * mmsr/models/archs/DCNv2/src/vision.cpp:3-8 (pybind export), src/dcn_v2.h:75-144 (dispatch),
 * src/cuda/dcn_v2_psroi_pooling_cuda.cu:58-419 (kernels and host side); called by dcn_v2.py:256-411.
 * Tensors are contiguous and all of one dtype T (f32 or f64 entry points):
 *   input [B,C,H,W]; bbox [R,5] rows (batch, x1, y1, x2, y2); trans [R, 2*num_classes, part_size, part_size]
 *   (unused and may be NULL when no_trans); out, count [R, output_dim, pooled_size, pooled_size].
 * ROI n: start = round(x1) * spatial_scale - 0.5, end = (round(x2) + 1) * spatial_scale - 0.5 (round half away from
 * zero), size = max(end - start, 0.1); bin (ph, pw) of size/pooled_size, S = sample_per_part samples per axis at
 *   start + p * bin + trans[n, cls, {0,1}, part(ph), part(pw)] * trans_std * size + i * bin / S,
 * part(p) = floor(T(p) / pooled_size * part_size), cls = c / (output_dim / num_classes).  A sample outside
 * [-0.5, W-0.5] x [-0.5, H-0.5] is dropped; a kept one is clamped to [0, W-1] x [0, H-1] and blends its floor / ceil
 * corners.  out = mean of the kept samples (0 if none), count = their number.  spatial_scale and trans_std are
 * float for both dtypes (as in the reference).
 * Rejected with C2M_ERR_INVALID (the reference reads out of bounds): C != output_dim, group_size != 1, num_classes
 * not dividing output_dim, pooled_size / part_size / sample_per_part < 1, sample_per_part > 45.  A batch index
 * int(bbox[n,0]) outside [0,B) gives out 0, count 0 and no gradient.
 * Backward: grad_input [B,C,H,W] is ACCUMULATED with atomics and grad_trans (shape of trans) is written in a fixed
 * summation order (bitwise reproducible); the caller zero-fills both.  Each gradient term is divided by top_count.
 * The workspace (c2m_psroi_pooling_workspace_bytes(shape, sizeof(T)) bytes, 0 when no_trans) holds one partial
 * trans gradient per output element. */
typedef struct {
    int B, C, H, W, R;
    int no_trans, num_classes;
    float spatial_scale, trans_std;
    int output_dim, group_size, pooled_size, part_size, sample_per_part;
} c2m_psroi_shape;

size_t c2m_psroi_pooling_workspace_bytes(const c2m_psroi_shape *shape, int elem_bytes);
int c2m_psroi_pooling_forward_f32(const float *input, const float *bbox, const float *trans,
                                  const c2m_psroi_shape *shape, float *out, float *count, c2m_stream_t stream);
int c2m_psroi_pooling_forward_f64(const double *input, const double *bbox, const double *trans,
                                  const c2m_psroi_shape *shape, double *out, double *count, c2m_stream_t stream);
int c2m_psroi_pooling_backward_f32(const float *out_grad, const float *input, const float *bbox, const float *trans,
                                   const float *top_count, const c2m_psroi_shape *shape, float *grad_input,
                                   float *grad_trans, void *ws, size_t ws_bytes, c2m_stream_t stream);
int c2m_psroi_pooling_backward_f64(const double *out_grad, const double *input, const double *bbox,
                                   const double *trans, const double *top_count, const c2m_psroi_shape *shape,
                                   double *grad_input, double *grad_trans, void *ws, size_t ws_bytes,
                                   c2m_stream_t stream);

/* ordered PS-ROI grad_input: see "ordered input gradients" above */
size_t c2m_psroi_grad_input_det_workspace_bytes(const c2m_psroi_shape *shape, int planes);
int c2m_psroi_pooling_grad_input_det_f32(const float *out_grad, const float *bbox, const float *trans,
                                         const float *top_count, const c2m_psroi_shape *shape, float *grad_input,
                                         void *ws, size_t ws_bytes, c2m_stream_t stream);
int c2m_psroi_pooling_grad_input_det_f64(const double *out_grad, const double *bbox, const double *trans,
                                         const double *top_count, const c2m_psroi_shape *shape, double *grad_input,
                                         void *ws, size_t ws_bytes, c2m_stream_t stream);

/* number of kernels this library has launched since load (bench.py's gpu_launches) */
unsigned long long c2m_launch_count(void);

/* Measurement hook (bench.py `roofline`): while enabled, the library brackets every launch of its
 * heavy kernel classes with CUDA events on the caller's stream:
 *   0 = correlation candidate search (corr_umma / generic), 1 = conv3x3_umma, 2 = dcn_umma,
 *   3 = c2m_dcn_tc_dgrad, 4 = c2m_dcn_tc_wgrad (with its reduce).
 * c2m_profile_collect synchronises the recorded events of one class, returns their summed device
 * time, launch count and summed ALGORITHMIC flops / bytes (SURVEY.md §8d formulas), and clears them. */
int c2m_profile_enable(int on);
int c2m_profile_collect(int kernel, float *ms_total, int *launches, double *flops, double *bytes);

#ifdef __cplusplus
}
#endif
#endif /* C2M_SM100_H */
