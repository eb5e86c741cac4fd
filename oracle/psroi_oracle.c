/*
 * ORACLE — test infrastructure, NOT product code.
 *
 * Plain-C, literal CPU restatement of deformable PS-ROI pooling, forward and backward, for float and double
 * (`_ext.dcn_v2_psroi_pooling_forward` / `_backward`; semantics of
 * DCNv2/src/cuda/dcn_v2_psroi_pooling_cuda.cu:58-269, host side :271-419).  One loop iteration per output element
 * (n, ctop, ph, pw), as the reference's kernels are written; only tests/ and tools/ load the library built from this
 * file (oracle/psroi_oracle.py).
 *
 * Arithmetic: every position is computed in T with the reference's expressions and promotions (a float minus the
 * double 0.5 is rounded back to float, max(size, 0.1) compares against the double 0.1, the skip test and the clamp
 * run in double).  The bilinear values, the per-bin sums and every gradient accumulate in double and are rounded to
 * T once.  Built with -ffp-contract=off, so no multiply-add is fused.
 *
 * Deliberate differences from the reference (which reads out of bounds in each case): the rejected arguments return
 * 1; a batch index outside [0, B) after truncation gives output 0, count 0 and no gradient.
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared -o oracle/_build/libpsroi_oracle.so oracle/psroi_oracle.c -lm
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

static int psroi_bad_args(int C, int no_trans, int num_classes, int output_dim, int group_size, int pooled_size,
                          int part_size, int sample_per_part)
{
    if (C != output_dim || group_size != 1) return 1;
    if (pooled_size < 1 || part_size < 1 || sample_per_part < 1) return 1;
    if (!no_trans && (num_classes < 1 || output_dim % num_classes)) return 1;
    return 0;
}

/* Geometry shared by the forward and backward bodies: declares roi_batch_ind, roi_width / roi_height, part_h / part_w,
 * class_id, wstart / hstart and sub_bin_size_w / _h for output element `index`, exactly as the reference's kernels. */
#define PSROI_GEOMETRY(T, ROUND)                                                                                    \
    const int pw = (int)(index % pooled_size);                                                                      \
    const int ph = (int)((index / pooled_size) % pooled_size);                                                      \
    const int ctop = (int)((index / pooled_size / pooled_size) % output_dim);                                       \
    const long n = index / pooled_size / pooled_size / output_dim;                                                  \
    const T *offset_bottom_rois = bbox + n * 5;                                                                     \
    const int roi_batch_ind = (int)offset_bottom_rois[0];                                                           \
    const T roi_start_w = (T)(ROUND(offset_bottom_rois[1])) * spatial_scale - 0.5;                                  \
    const T roi_start_h = (T)(ROUND(offset_bottom_rois[2])) * spatial_scale - 0.5;                                  \
    const T roi_end_w = (T)(ROUND(offset_bottom_rois[3]) + 1.) * spatial_scale - 0.5;                               \
    const T roi_end_h = (T)(ROUND(offset_bottom_rois[4]) + 1.) * spatial_scale - 0.5;                               \
    const T roi_width = fmax(roi_end_w - roi_start_w, 0.1);                                                         \
    const T roi_height = fmax(roi_end_h - roi_start_h, 0.1);                                                        \
    const T bin_size_h = roi_height / (T)pooled_size;                                                               \
    const T bin_size_w = roi_width / (T)pooled_size;                                                                \
    const T sub_bin_size_h = bin_size_h / (T)sample_per_part;                                                       \
    const T sub_bin_size_w = bin_size_w / (T)sample_per_part;                                                       \
    const int part_h = (int)floor((T)ph / pooled_size * part_size);                                                 \
    const int part_w = (int)floor((T)pw / pooled_size * part_size);                                                 \
    const int class_id = ctop / channels_each_class;                                                                \
    const long tx_i = (((n * num_classes + class_id) * 2) * part_size + part_h) * part_size + part_w;               \
    const long ty_i = (((n * num_classes + class_id) * 2 + 1) * part_size + part_h) * part_size + part_w;           \
    const T trans_x = no_trans ? (T)0 : trans[tx_i] * trans_std;                                                    \
    const T trans_y = no_trans ? (T)0 : trans[ty_i] * trans_std;                                                    \
    T wstart = (T)pw * bin_size_w + roi_start_w;                                                                    \
    wstart += trans_x * roi_width;                                                                                  \
    T hstart = (T)ph * bin_size_h + roi_start_h;                                                                    \
    hstart += trans_y * roi_height;                                                                                 \
    const int batch_ok = roi_batch_ind >= 0 && roi_batch_ind < B && H > 0 && W > 0

/* One sample (ih, iw): `continue`s when it is dropped, else declares the clamped corners and distances. */
#define PSROI_SAMPLE(T)                                                                                             \
    T w = wstart + iw * sub_bin_size_w;                                                                             \
    T h = hstart + ih * sub_bin_size_h;                                                                             \
    if (w < -0.5 || w > W - 0.5 || h < -0.5 || h > H - 0.5) continue;                                               \
    w = fmin(fmax(w, 0.), W - 1.);                                                                                  \
    h = fmin(fmax(h, 0.), H - 1.);                                                                                  \
    const int x0 = (int)floor(w), x1 = (int)ceil(w), y0 = (int)floor(h), y1 = (int)ceil(h);                        \
    const T dist_x = w - x0, dist_y = h - y0

#define DEFINE_PSROI(T, SFX, ROUND)                                                                                 \
int oracle_psroi_forward_##SFX(const T *input, const T *bbox, const T *trans, int B, int C, int H, int W, int R,    \
                               int no_trans, int num_classes, float spatial_scale_f, int output_dim,                \
                               int group_size, int pooled_size, int part_size, int sample_per_part,                 \
                               float trans_std_f, T *out, T *count)                                                 \
{                                                                                                                   \
    if (psroi_bad_args(C, no_trans, num_classes, output_dim, group_size, pooled_size, part_size, sample_per_part))  \
        return 1;                                                                                                   \
    const T spatial_scale = (T)spatial_scale_f, trans_std = (T)trans_std_f;                                         \
    if (no_trans) num_classes = 1;                                                                                  \
    const int channels_each_class = output_dim / num_classes;                                                       \
    const long total = (long)R * output_dim * pooled_size * pooled_size;                                            \
    for (long index = 0; index < total; ++index) {                                                                  \
        PSROI_GEOMETRY(T, ROUND);                                                                                   \
        double sum = 0.0;                                                                                           \
        int cnt = 0;                                                                                                \
        if (batch_ok) {                                                                                             \
            const T *im = input + ((long)roi_batch_ind * C + ctop) * H * W;                                         \
            for (int ih = 0; ih < sample_per_part; ih++) {                                                          \
                for (int iw = 0; iw < sample_per_part; iw++) {                                                      \
                    PSROI_SAMPLE(T);                                                                                \
                    const double dx = dist_x, dy = dist_y;                                                          \
                    sum += (1 - dx) * (1 - dy) * im[y0 * W + x0] + (1 - dx) * dy * im[y1 * W + x0] +                \
                           dx * (1 - dy) * im[y0 * W + x1] + dx * dy * im[y1 * W + x1];                             \
                    cnt++;                                                                                          \
                }                                                                                                   \
            }                                                                                                       \
        }                                                                                                           \
        out[index] = cnt == 0 ? (T)0 : (T)(sum / cnt);                                                              \
        count[index] = (T)cnt;                                                                                      \
    }                                                                                                               \
    return 0;                                                                                                       \
}                                                                                                                   \
                                                                                                                    \
int oracle_psroi_backward_##SFX(const T *top_diff, const T *input, const T *bbox, const T *trans,                   \
                                const T *top_count, int B, int C, int H, int W, int R, int no_trans,                \
                                int num_classes, float spatial_scale_f, int output_dim, int group_size,             \
                                int pooled_size, int part_size, int sample_per_part, float trans_std_f,             \
                                T *grad_input, T *grad_trans)                                                       \
{                                                                                                                   \
    if (psroi_bad_args(C, no_trans, num_classes, output_dim, group_size, pooled_size, part_size, sample_per_part))  \
        return 1;                                                                                                   \
    const T spatial_scale = (T)spatial_scale_f, trans_std = (T)trans_std_f;                                         \
    if (no_trans) num_classes = 1;                                                                                  \
    const int channels_each_class = output_dim / num_classes;                                                       \
    const long total = (long)R * output_dim * pooled_size * pooled_size;                                            \
    const long n_in = (long)B * C * H * W, n_tr = no_trans ? 0 : (long)R * 2 * num_classes * part_size * part_size; \
    double *gin = (double *)calloc(n_in ? n_in : 1, sizeof(double));                                                \
    double *gtr = (double *)calloc(n_tr ? n_tr : 1, sizeof(double));                                                \
    if (!gin || !gtr) { free(gin); free(gtr); return 2; }                                                           \
    for (long index = 0; index < total; ++index) {                                                                  \
        PSROI_GEOMETRY(T, ROUND);                                                                                   \
        if (!batch_ok || top_count[index] <= 0) continue;                                                           \
        const double diff_val = (double)top_diff[index] / top_count[index];                                         \
        const T *im = input + ((long)roi_batch_ind * C + ctop) * H * W;                                             \
        double *gim = gin + ((long)roi_batch_ind * C + ctop) * H * W;                                               \
        for (int ih = 0; ih < sample_per_part; ih++) {                                                              \
            for (int iw = 0; iw < sample_per_part; iw++) {                                                          \
                PSROI_SAMPLE(T);                                                                                    \
                const double dx = dist_x, dy = dist_y;                                                              \
                gim[y0 * W + x0] += (1 - dx) * (1 - dy) * diff_val;                                                 \
                gim[y1 * W + x0] += (1 - dx) * dy * diff_val;                                                       \
                gim[y0 * W + x1] += dx * (1 - dy) * diff_val;                                                       \
                gim[y1 * W + x1] += dx * dy * diff_val;                                                             \
                if (no_trans) continue;                                                                             \
                const double U00 = im[y0 * W + x0], U01 = im[y1 * W + x0];                                          \
                const double U10 = im[y0 * W + x1], U11 = im[y1 * W + x1];                                          \
                gtr[tx_i] += (U11 * dy + U10 * (1 - dy) - U01 * dy - U00 * (1 - dy)) * trans_std * diff_val *       \
                             roi_width;                                                                             \
                gtr[ty_i] += (U11 * dx + U01 * (1 - dx) - U10 * dx - U00 * (1 - dx)) * trans_std * diff_val *       \
                             roi_height;                                                                            \
            }                                                                                                       \
        }                                                                                                           \
    }                                                                                                               \
    for (long i = 0; i < n_in; ++i) grad_input[i] = (T)gin[i];                                                      \
    for (long i = 0; i < n_tr; ++i) grad_trans[i] = (T)gtr[i];                                                      \
    free(gin);                                                                                                      \
    free(gtr);                                                                                                      \
    return 0;                                                                                                       \
}

DEFINE_PSROI(float, f32, roundf)
DEFINE_PSROI(double, f64, round)
