/*
 * ORACLE — test infrastructure, NOT product code.
 *
 * Plain-C, literal CPU restatement of grouped deformable convolution, v1 (no mask) and modulated, forward and
 * backward, for float and double: the semantics of the reference's `deform_conv_cuda` extension
 * (dcn/src/deform_conv_cuda.cpp:151-679 host side; deformable_im2col / col2im / col2im_coord and the modulated
 * kernels in dcn/src/deform_conv_cuda_kernel.cu).  Only tests/ and tools/ load the library built from this file
 * (oracle/deform_conv_oracle.py).  oracle/c2m_oracle.c keeps the fp32 `_ext` restatement the older tests pin.
 *
 *   out[b,o,p] = bias[o] + sum_{cl < C/groups, i, j} W[o,cl,i,j] * m * bilinear(x[b,c], h_im, w_im)
 *   c = (o / (Cout/groups)) * (C/groups) + cl        (conv group of o)
 *   h_im = ho*sh - ph + i*dh + offset[b, 2*(g*kh*kw + i*kw + j)    , p],  g = c / (C/dg)  (deformable group of c)
 *   w_im = wo*sw - pw + j*dw + offset[b, 2*(g*kh*kw + i*kw + j) + 1, p]
 *   m = mask[b, g*kh*kw + i*kw + j, p], or 1 when mask is NULL (v1); the sample is 0 unless -1 < h_im < H, -1 < w_im < W
 *
 * Arithmetic: positions and the bilinear column value are computed in T in the order of the reference's `scalar_t`
 * kernels (float positions for f32, as oracle_dcn_v2_* in c2m_oracle.c); the contraction, the bias add and every
 * gradient accumulate in double and are rounded to T once.  With groups == 1 and a mask, the f32 instantiation is
 * oracle_dcn_v2_forward (acc64) / oracle_dcn_v2_backward bit for bit.  Built with -ffp-contract=off.
 *
 * Build: gcc -O2 -fopenmp -ffp-contract=off -fPIC -shared -o oracle/_build/libdeform_conv_oracle.so \
 *        oracle/deform_conv_oracle.c -lm
 */
#include <math.h>
#include <stdlib.h>

static int deform_bad_args(int C, int Cout, int groups, int dg, int Ho, int Wo)
{
    if (groups < 1 || C % groups || Cout % groups) return 1;
    if (dg < 1 || C % dg) return 1;
    return Ho < 1 || Wo < 1;
}

#define DEFINE_DEFORM_CONV(T, SFX, FLOOR)                                                                           \
static T bilinear_##SFX(const T *im, int H, int W, T h, T w)                                                        \
{                                                                                                                   \
    int h_low = (int)FLOOR(h), w_low = (int)FLOOR(w);                                                               \
    int h_high = h_low + 1, w_high = w_low + 1;                                                                     \
    T lh = h - h_low, lw = w - w_low;                                                                               \
    T hh = 1 - lh, hw = 1 - lw;                                                                                     \
    T v1 = 0, v2 = 0, v3 = 0, v4 = 0;                                                                               \
    if (h_low >= 0 && w_low >= 0) v1 = im[h_low * W + w_low];                                                       \
    if (h_low >= 0 && w_high <= W - 1) v2 = im[h_low * W + w_high];                                                 \
    if (h_high <= H - 1 && w_low >= 0) v3 = im[h_high * W + w_low];                                                 \
    if (h_high <= H - 1 && w_high <= W - 1) v4 = im[h_high * W + w_high];                                           \
    T w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;                                                       \
    return (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);                                                                 \
}                                                                                                                   \
                                                                                                                    \
int oracle_deform_conv_forward_##SFX(const T *x, const T *weight, const T *bias, const T *offset, const T *mask,     \
                                     T *out, int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw,  \
                                     int ph, int pw, int dh, int dw, int groups, int dg)                            \
{                                                                                                                   \
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;                                                     \
    const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;                                                     \
    if (deform_bad_args(C, Cout, groups, dg, Ho, Wo)) return 1;                                                     \
    const int T_ = kh * kw, K = C * T_, cpg = C / dg, Kg = K / groups, cout_g = Cout / groups;                      \
    const long P = (long)Ho * Wo;                                                                                   \
    int fail = 0;                                                                                                   \
    _Pragma("omp parallel")                                                                                         \
    {                                                                                                               \
        T *col = (T *)malloc(sizeof(T) * K);                                                                        \
        if (!col) fail = 1;                                                                                         \
        _Pragma("omp for collapse(2) schedule(static)")                                                             \
        for (int b = 0; b < B; ++b)                                                                                 \
            for (long p = 0; p < P; ++p) {                                                                          \
                if (!col) continue;                                                                                 \
                const int ho = (int)(p / Wo), wo = (int)(p % Wo);                                                   \
                const int h_in = ho * sh - ph, w_in = wo * sw - pw;                                                 \
                for (int c = 0; c < C; ++c) {                                                                       \
                    const int g = c / cpg;                                                                          \
                    const T *im = x + ((long)b * C + c) * H * W;                                                    \
                    const T *offp = offset + ((long)b * dg + g) * 2 * T_ * P;                                       \
                    for (int i = 0; i < kh; ++i)                                                                    \
                        for (int j = 0; j < kw; ++j) {                                                              \
                            const int k = i * kw + j;                                                               \
                            const T oh = offp[(long)(2 * k) * P + p];                                               \
                            const T ow = offp[(long)(2 * k + 1) * P + p];                                           \
                            const T m = mask ? mask[(((long)b * dg + g) * T_ + k) * P + p] : (T)1;                  \
                            const T h_im = h_in + i * dh + oh;                                                      \
                            const T w_im = w_in + j * dw + ow;                                                      \
                            T v = 0;                                                                                \
                            if (h_im > -1 && w_im > -1 && h_im < H && w_im < W)                                     \
                                v = bilinear_##SFX(im, H, W, h_im, w_im);                                           \
                            col[(c * kh + i) * kw + j] = v * m;                                                     \
                        }                                                                                           \
                }                                                                                                   \
                for (int o = 0; o < Cout; ++o) {                                                                    \
                    const T *wrow = weight + (long)o * Kg;                                                          \
                    const T *crow = col + (long)(o / cout_g) * Kg;                                                  \
                    double acc = 0.0;                                                                               \
                    for (int k = 0; k < Kg; ++k) acc += (double)wrow[k] * (double)crow[k];                          \
                    out[((long)b * Cout + o) * P + p] = (T)(acc + (double)(bias ? bias[o] : (T)0));                 \
                }                                                                                                   \
            }                                                                                                       \
        free(col);                                                                                                  \
    }                                                                                                               \
    return fail ? 2 : 0;                                                                                            \
}                                                                                                                   \
                                                                                                                    \
/* gcol[b, c*T+k, p] = sum over the conv group's o of W[o, cl*T+k] * gout[b,o,p]; then, per deformable group:         \
 *   grad_mask   = sum_{c in g} gcol * bilinear                       (only when mask != NULL)                       \
 *   grad_offset = sum_{c in g} gcol * m * d bilinear / d h|w                                                        \
 *   grad_input += gcol * m * corner weight, in-image corners only                                                   \
 *   grad_weight[o, cl*T+k] = sum_{b,p} gout[b,o,p] * m * bilinear;  grad_bias[o] = sum_{b,p} gout[b,o,p] */         \
int oracle_deform_conv_backward_##SFX(const T *x, const T *weight, const T *offset, const T *mask, const T *gout,    \
                                      T *gx, T *goff, T *gmask, T *gw, T *gb, int B, int C, int H, int W, int Cout, \
                                      int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int groups,   \
                                      int dg)                                                                       \
{                                                                                                                   \
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;                                                     \
    const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;                                                     \
    if (deform_bad_args(C, Cout, groups, dg, Ho, Wo)) return 1;                                                     \
    const int T_ = kh * kw, cpg = C / dg, cin_g = C / groups, cout_g = Cout / groups, Kg = cin_g * T_;              \
    const long P = (long)Ho * Wo;                                                                                   \
    double *dgx = (double *)calloc((size_t)B * C * H * W, sizeof(double));                                          \
    double *dgw = (double *)calloc((size_t)Cout * Kg, sizeof(double));                                              \
    double *dgb = (double *)calloc((size_t)Cout, sizeof(double));                                                   \
    if (!dgx || !dgw || !dgb) { free(dgx); free(dgw); free(dgb); return 2; }                                        \
    for (int b = 0; b < B; ++b)                                                                                     \
        for (long p = 0; p < P; ++p) {                                                                              \
            const int ho = (int)(p / Wo), wo = (int)(p % Wo);                                                       \
            for (int o = 0; o < Cout; ++o) dgb[o] += gout[((long)b * Cout + o) * P + p];                            \
            for (int g = 0; g < dg; ++g)                                                                            \
                for (int k = 0; k < T_; ++k) {                                                                      \
                    const int i = k / kw, j = k % kw;                                                               \
                    const T oh = offset[(((long)b * dg + g) * 2 * T_ + 2 * k) * P + p];                             \
                    const T ow = offset[(((long)b * dg + g) * 2 * T_ + 2 * k + 1) * P + p];                         \
                    const T m = mask ? mask[(((long)b * dg + g) * T_ + k) * P + p] : (T)1;                          \
                    const T h_im = (T)(ho * sh - ph + i * dh) + oh;                                                 \
                    const T w_im = (T)(wo * sw - pw + j * dw) + ow;                                                 \
                    const int valid = h_im > -1 && w_im > -1 && h_im < H && w_im < W;                               \
                    double acc_h = 0, acc_w = 0, acc_m = 0;                                                         \
                    const int hl = (int)FLOOR(h_im), wl = (int)FLOOR(w_im), hh_ = hl + 1, wh = wl + 1;              \
                    const double lh = (double)h_im - hl, lw = (double)w_im - wl;                                    \
                    for (int cl = 0; cl < cpg; ++cl) {                                                              \
                        const int c = g * cpg + cl, cg = c / cin_g, ck = (c - cg * cin_g) * T_ + k;                 \
                        double gc = 0;                                                                              \
                        for (int o = cg * cout_g; o < (cg + 1) * cout_g; ++o)                                       \
                            gc += (double)weight[(long)o * Kg + ck] * gout[((long)b * Cout + o) * P + p];           \
                        const T *im = x + ((long)b * C + c) * H * W;                                                \
                        double v1 = 0, v2 = 0, v3 = 0, v4 = 0;                                                      \
                        if (valid) {                                                                                \
                            if (hl >= 0 && wl >= 0) v1 = im[hl * W + wl];                                           \
                            if (hl >= 0 && wh <= W - 1) v2 = im[hl * W + wh];                                       \
                            if (hh_ <= H - 1 && wl >= 0) v3 = im[hh_ * W + wl];                                     \
                            if (hh_ <= H - 1 && wh <= W - 1) v4 = im[hh_ * W + wh];                                 \
                        }                                                                                           \
                        const double val = (1 - lh) * (1 - lw) * v1 + (1 - lh) * lw * v2 + lh * (1 - lw) * v3 +     \
                                           lh * lw * v4;                                                            \
                        const double col = valid ? val * m : 0.0;                                                   \
                        for (int o = cg * cout_g; o < (cg + 1) * cout_g; ++o)                                       \
                            dgw[(long)o * Kg + ck] += (double)gout[((long)b * Cout + o) * P + p] * col;             \
                        if (valid) {                                                                                \
                            acc_m += gc * val;                                                                      \
                            acc_h += gc * m * (-(1 - lw) * v1 - lw * v2 + (1 - lw) * v3 + lw * v4);                 \
                            acc_w += gc * m * (-(1 - lh) * v1 + (1 - lh) * v2 - lh * v3 + lh * v4);                 \
                            const double tg = gc * m;                                                               \
                            double *gim = dgx + ((long)b * C + c) * H * W;                                          \
                            if (hl >= 0 && wl >= 0) gim[hl * W + wl] += tg * (1 - lh) * (1 - lw);                   \
                            if (hl >= 0 && wh <= W - 1) gim[hl * W + wh] += tg * (1 - lh) * lw;                     \
                            if (hh_ <= H - 1 && wl >= 0) gim[hh_ * W + wl] += tg * lh * (1 - lw);                   \
                            if (hh_ <= H - 1 && wh <= W - 1) gim[hh_ * W + wh] += tg * lh * lw;                     \
                        }                                                                                           \
                    }                                                                                               \
                    goff[(((long)b * dg + g) * 2 * T_ + 2 * k) * P + p] = (T)acc_h;                                 \
                    goff[(((long)b * dg + g) * 2 * T_ + 2 * k + 1) * P + p] = (T)acc_w;                             \
                    if (mask) gmask[(((long)b * dg + g) * T_ + k) * P + p] = (T)acc_m;                              \
                }                                                                                                   \
        }                                                                                                           \
    for (long i = 0; i < (long)B * C * H * W; ++i) gx[i] = (T)dgx[i];                                               \
    for (long i = 0; i < (long)Cout * Kg; ++i) gw[i] = (T)dgw[i];                                                   \
    for (int o = 0; o < Cout; ++o) gb[o] = (T)dgb[o];                                                               \
    free(dgx); free(dgw); free(dgb);                                                                                \
    return 0;                                                                                                       \
}

DEFINE_DEFORM_CONV(float, f32, floorf)
DEFINE_DEFORM_CONV(double, f64, floor)
