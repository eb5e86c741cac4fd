/*
 * ORACLE — test infrastructure, NOT product code.
 *
 * Plain-C restatement of the ordered input gradients of deformable convolution and deformable PS-ROI pooling, in the
 * dtype, for float and double: the sums the c2m_*_det entry points of include/c2m_sm100.h compute when torch's
 * deterministic algorithms are enabled.  Every element of grad_input starts at +0 and adds its contributions in T,
 * one correctly rounded add each, in this order:
 *
 *   DCN: ascending tap k, then output pixel p, then corner (low-low, low-high, high-low, high-high); a contribution is
 *        ((gcol * m) * hh) * hw and so on (m = 1 without a mask), in-image corners of in-window points only.
 *   PS-ROI: ascending ROI n, then bin (ph, pw) row-major, then sample (ih, iw) row-major, then corner (floor, +dy, +dx,
 *        +dx+dy); a contribution is (hx * hy) * diff and so on with diff = out_grad / count; dropped samples, ROIs with
 *        an invalid batch index, count <= 0 and corners that coincide with the floor corner contribute nothing.
 *
 * Looping over (k, p, corner), resp. (n, channel, bin, sample, corner), and adding into each element as it comes gives
 * every element its contributions in that order.  Positions are computed as in oracle/deform_conv_oracle.c and
 * oracle/psroi_oracle.c.  They take gcol (resp. out_grad and top_count) as given.  Only tests/ and tools/ load the
 * library built from this file (oracle/ordered_grad_oracle.py).
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared -o oracle/_build/libordered_grad_oracle.so \
 *        oracle/ordered_grad_oracle.c -lm
 */
#include <math.h>
#include <string.h>

#define DEFINE_ORDERED(T, SFX, FLOOR, ROUND)                                                                        \
int oracle_deform_col2im_ordered_##SFX(const T *gcol, const T *offset, const T *mask, T *gx, int B, int C, int H,   \
                                       int W, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,        \
                                       int dg)                                                                      \
{                                                                                                                   \
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;                                                     \
    const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;                                                     \
    if (dg < 1 || C % dg || Ho < 1 || Wo < 1) return 1;                                                             \
    const int T_ = kh * kw, cpg = C / dg;                                                                           \
    const long P = (long)Ho * Wo;                                                                                   \
    for (long i = 0; i < (long)B * C * H * W; ++i) gx[i] = (T)0;                                                    \
    for (int b = 0; b < B; ++b)                                                                                     \
        for (int c = 0; c < C; ++c) {                                                                               \
            const int g = c / cpg;                                                                                  \
            T *gim = gx + ((long)b * C + c) * H * W;                                                                \
            for (int k = 0; k < T_; ++k)                                                                            \
                for (long p = 0; p < P; ++p) {                                                                      \
                    const int i = k / kw, j = k % kw, ho = (int)(p / Wo), wo = (int)(p % Wo);                       \
                    const long jj = ((long)b * dg + g) * T_ + k;                                                    \
                    const T h_im = (T)(ho * sh - ph + i * dh) + offset[2 * jj * P + p];                             \
                    const T w_im = (T)(wo * sw - pw + j * dw) + offset[(2 * jj + 1) * P + p];                       \
                    if (!(h_im > -1 && w_im > -1 && h_im < H && w_im < W)) continue;                                \
                    const int hl = (int)FLOOR(h_im), wl = (int)FLOOR(w_im), hh_ = hl + 1, wh = wl + 1;              \
                    const T lh = h_im - hl, lw = w_im - wl, hh = (T)1 - lh, hw = (T)1 - lw;                         \
                    const T tg = gcol[(((long)b * C + c) * T_ + k) * P + p] * (mask ? mask[jj * P + p] : (T)1);     \
                    if (hl >= 0 && wl >= 0) gim[hl * W + wl] += tg * hh * hw;                                       \
                    if (hl >= 0 && wh <= W - 1) gim[hl * W + wh] += tg * hh * lw;                                   \
                    if (hh_ <= H - 1 && wl >= 0) gim[hh_ * W + wl] += tg * lh * hw;                                 \
                    if (hh_ <= H - 1 && wh <= W - 1) gim[hh_ * W + wh] += tg * lh * lw;                             \
                }                                                                                                   \
        }                                                                                                           \
    return 0;                                                                                                       \
}                                                                                                                   \
                                                                                                                    \
int oracle_psroi_grad_input_ordered_##SFX(const T *top_diff, const T *bbox, const T *trans, const T *top_count,     \
                                          int B, int C, int H, int W, int R, int no_trans, int num_classes,         \
                                          float spatial_scale_f, int output_dim, int group_size, int pooled_size,   \
                                          int part_size, int sample_per_part, float trans_std_f, T *grad_input)     \
{                                                                                                                   \
    if (C != output_dim || group_size != 1 || pooled_size < 1 || part_size < 1 || sample_per_part < 1) return 1;    \
    if (!no_trans && (num_classes < 1 || output_dim % num_classes)) return 1;                                       \
    const T spatial_scale = (T)spatial_scale_f, trans_std = (T)trans_std_f;                                         \
    if (no_trans) num_classes = 1;                                                                                  \
    const int channels_each_class = output_dim / num_classes;                                                       \
    for (long i = 0; i < (long)B * C * H * W; ++i) grad_input[i] = (T)0;                                            \
    for (long n = 0; n < R; ++n)                                                                                    \
        for (int ctop = 0; ctop < output_dim; ++ctop)                                                               \
            for (int ph = 0; ph < pooled_size; ++ph)                                                                \
                for (int pw = 0; pw < pooled_size; ++pw) {                                                          \
                    const long index = ((n * output_dim + ctop) * pooled_size + ph) * pooled_size + pw;             \
                    const T *roi = bbox + n * 5;                                                                    \
                    const int b = (int)roi[0];                                                                      \
                    if (!(b >= 0 && b < B && H > 0 && W > 0) || top_count[index] <= 0) continue;                   \
                    const T start_w = (T)(ROUND(roi[1])) * spatial_scale - 0.5;                                     \
                    const T start_h = (T)(ROUND(roi[2])) * spatial_scale - 0.5;                                     \
                    const T end_w = (T)(ROUND(roi[3]) + 1.) * spatial_scale - 0.5;                                  \
                    const T end_h = (T)(ROUND(roi[4]) + 1.) * spatial_scale - 0.5;                                  \
                    const T roi_w = fmax(end_w - start_w, 0.1), roi_h = fmax(end_h - start_h, 0.1);                 \
                    const T bin_h = roi_h / (T)pooled_size, bin_w = roi_w / (T)pooled_size;                         \
                    const T sub_h = bin_h / (T)sample_per_part, sub_w = bin_w / (T)sample_per_part;                 \
                    const int part_h = (int)floor((T)ph / pooled_size * part_size);                                 \
                    const int part_w = (int)floor((T)pw / pooled_size * part_size);                                 \
                    const int cls = ctop / channels_each_class;                                                     \
                    const long tx_i = (((n * num_classes + cls) * 2) * part_size + part_h) * part_size + part_w;    \
                    const long ty_i = (((n * num_classes + cls) * 2 + 1) * part_size + part_h) * part_size + part_w; \
                    const T trans_x = no_trans ? (T)0 : trans[tx_i] * trans_std;                                    \
                    const T trans_y = no_trans ? (T)0 : trans[ty_i] * trans_std;                                    \
                    T wstart = (T)pw * bin_w + start_w;                                                             \
                    wstart += trans_x * roi_w;                                                                      \
                    T hstart = (T)ph * bin_h + start_h;                                                             \
                    hstart += trans_y * roi_h;                                                                      \
                    const T diff = top_diff[index] / top_count[index];                                              \
                    T *gim = grad_input + ((long)b * C + ctop) * H * W;                                             \
                    for (int ih = 0; ih < sample_per_part; ++ih)                                                    \
                        for (int iw = 0; iw < sample_per_part; ++iw) {                                              \
                            T w = wstart + iw * sub_w;                                                              \
                            T h = hstart + ih * sub_h;                                                              \
                            if (w < -0.5 || w > W - 0.5 || h < -0.5 || h > H - 0.5) continue;                       \
                            w = fmin(fmax(w, 0.), W - 1.);                                                          \
                            h = fmin(fmax(h, 0.), H - 1.);                                                          \
                            const int x0 = (int)floor(w), x1 = (int)ceil(w), y0 = (int)floor(h), y1 = (int)ceil(h); \
                            const T lx = w - x0, ly = h - y0, hx = (T)1 - lx, hy = (T)1 - ly;                       \
                            gim[y0 * W + x0] += hx * hy * diff;                                                     \
                            if (y1 != y0) gim[y1 * W + x0] += hx * ly * diff;                                       \
                            if (x1 != x0) gim[y0 * W + x1] += lx * hy * diff;                                       \
                            if (x1 != x0 && y1 != y0) gim[y1 * W + x1] += lx * ly * diff;                           \
                        }                                                                                           \
                }                                                                                                   \
    return 0;                                                                                                       \
}

DEFINE_ORDERED(float, f32, floorf, roundf)
DEFINE_ORDERED(double, f64, floor, round)
