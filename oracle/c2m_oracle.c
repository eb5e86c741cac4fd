/*
 * ORACLE — test infrastructure, NOT product code.
 *
 * Plain-C, literal CPU restatement of the two kernels of the C2-Matching restoration-forward
 * hot path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load
 * the library built from this file (oracle/c_oracle.py); nothing under c2-matching_b200/ does.
 *
 * Parity status: PINNED — tests/test_oracle.py checks every entry point against
 * tests/golden/*.npz, which were minted from the unmodified reference Python run on CPU
 * (tests/golden/make_golden.py).  The reference ships no golden vectors of its own.
 *
 * Citations are relative to /root/reference/mmsr/models/archs/.
 *
 * Build: gcc -O2 -fopenmp -fPIC -shared -o oracle/_build/libc2m_oracle.so oracle/c2m_oracle.c -lm
 * (-ffast-math is deliberately NOT used: summation order below is the documented one.)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * feature_match_index — ref_map_util.py:26-86
 *
 *   for each input patch q (row-major over the (h-p)/s_in+1 x (w-p)/s_in+1 grid):
 *     score(q, r) = < P_in(q), P_ref(r) / (||P_ref(r)||_2 + 1e-5) >        (:62-67)
 *     idx(q) = argmax_r score, lowest r on ties (first max within a chunk :69, strict '>'
 *              across chunks :74-76  =>  globally the lowest index among equal maxima)
 *              with torch's `max` rule for NaN: a NaN score is the maximum, the lowest-index NaN
 *              wins and val is NaN; +Inf is an ordinary maximum.  (The reference's strict '>'
 *              merge across chunks of 2^29 / (h*w) Ref patches makes NaN chunk-dependent once
 *              NR*h*w > 2^29; this oracle is the single-chunk rule.)
 *     val(q) = max_r score, divided by (||P_in(q)||_2 + 1e-5) if norm_input  (:78-84)
 *
 * Arithmetic: the reference normalises the Ref patches in fp32 BEFORE the dot product
 * (:63) — reproduced (each normalised element is rounded to float).  The dot product is
 * accumulated in double over (c, dy, dx) and rounded to float once, so this oracle is at
 * least as accurate as any fp32 summation order the reference's conv2d backend may pick;
 * `gap` receives the double-precision top-1 minus top-2 score per query so tests can tell
 * a genuine mismatch from a sub-ulp tie.
 * ------------------------------------------------------------------------------------------ */
int oracle_corr_argmax(const float *fin, const float *fref, int C, int h, int w, int hr, int wr,
                       int patch, int s_in, int s_ref, int is_norm, int norm_input,
                       int64_t *idx, float *val, double *gap /* may be NULL */)
{
    if (h < patch || w < patch || hr < patch || wr < patch) return 1;
    const int nh = (h - patch) / s_in + 1, nw = (w - patch) / s_in + 1;
    const int rh = (hr - patch) / s_ref + 1, rw = (wr - patch) / s_ref + 1;
    const int K = C * patch * patch;
    const long NR = (long)rh * rw, NQ = (long)nh * nw;

    /* materialised, normalised Ref patches [NR][K], K ordered (c, dy, dx) like conv2d weights */
    float *pref = (float *)malloc(sizeof(float) * NR * K);
    if (!pref) return 2;
#pragma omp parallel for schedule(static)
    for (long r = 0; r < NR; ++r) {
        const int ry = (int)(r / rw) * s_ref, rx = (int)(r % rw) * s_ref;
        float *p = pref + r * K;
        double ss = 0.0;
        for (int c = 0; c < C; ++c)
            for (int dy = 0; dy < patch; ++dy)
                for (int dx = 0; dx < patch; ++dx) {
                    float v = fref[((long)c * hr + ry + dy) * wr + rx + dx];
                    p[(c * patch + dy) * patch + dx] = v;
                    ss += (double)v * v;
                }
        if (is_norm) {
            const float denom = (float)sqrt(ss) + 1e-5f;        /* :63 */
            for (int k = 0; k < K; ++k) p[k] = p[k] / denom;
        }
    }

#pragma omp parallel
    {
        float *pq = (float *)malloc(sizeof(float) * K);
#pragma omp for schedule(dynamic, 4)
        for (long q = 0; q < NQ; ++q) {
            const int qy = (int)(q / nw) * s_in, qx = (int)(q % nw) * s_in;
            double ssq = 0.0;
            for (int c = 0; c < C; ++c)
                for (int dy = 0; dy < patch; ++dy)
                    for (int dx = 0; dx < patch; ++dx) {
                        float v = fin[((long)c * h + qy + dy) * w + qx + dx];
                        pq[(c * patch + dy) * patch + dx] = v;
                        ssq += (double)v * v;
                    }
            float best = -INFINITY;
            long besti = 0;
            double best_d = -INFINITY, second_d = -INFINITY;
            for (long r = 0; r < NR; ++r) {
                const float *p = pref + r * K;
                double acc = 0.0;
                for (int k = 0; k < K; ++k) acc += (double)pq[k] * (double)p[k];
                const float s = (float)acc;
                /* torch's max: NaN is the maximum (the first NaN wins), otherwise strict '>' => lowest index */
                if (!isnan(best) && (isnan(s) || s > best)) { best = s; besti = r; }
                if (acc > best_d) { second_d = best_d; best_d = acc; }
                else if (acc > second_d) second_d = acc;
            }
            idx[q] = besti;
            val[q] = norm_input ? best / ((float)sqrt(ssq) + 1e-5f) : best;   /* :78-84 */
            if (gap) gap[q] = best_d - second_d;
        }
        free(pq);
    }
    free(pref);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * index_to_flow + 9-shift x 3-scale pyramid — corres_generation_arch.py:29-46, 70-104;
 * tensor_shift arch_util.py:291-315.
 *
 *   flow[y][x] = (idx % gw - x, idx / gw - y) on the (gh x gw) patch grid, zero-padded by 2 at
 *   the bottom/right to (H x W) = (gh+2 x gw+2)                                   (:29-46)
 *   scale s in {1,2,4}: F_s[Y][X] = s * flow[Y/s][X/s]   (repeat_interleave, :84-87, :96-99)
 *   tap k = 3i+j: out_s[k][Y][X] = (Y >= s*i && X >= s*j) ? F_s[Y - s*i][X - s*j] : 0
 *
 * NB the reference decodes idx with the INPUT grid width gw (:32-34); `ref_gw` lets callers
 * that match against a differently sized Ref grid decode with the Ref width instead
 * (pass ref_gw = gw for reference behaviour).
 * out layout: [9][s*H][s*W][2] float, last dim (x, y).
 * ------------------------------------------------------------------------------------------ */
int oracle_offset_pyramid(const int64_t *idx, int gh, int gw, int ref_gw, int s, float *out)
{
    const int H = gh + 2, W = gw + 2, HS = H * s, WS = W * s;
    for (int k = 0; k < 9; ++k) {
        const int i = k / 3, j = k % 3;
        for (int Y = 0; Y < HS; ++Y)
            for (int X = 0; X < WS; ++X) {
                float fx = 0.f, fy = 0.f;
                const int ys = Y - s * i, xs = X - s * j;
                if (ys >= 0 && xs >= 0) {
                    const int y = ys / s, x = xs / s;
                    if (y < gh && x < gw) {
                        const int64_t v = idx[(long)y * gw + x];
                        fx = (float)(s * ((int)(v % ref_gw) - x));
                        fy = (float)(s * ((int)(v / ref_gw) - y));
                    }
                }
                float *o = out + (((long)k * HS + Y) * WS + X) * 2;
                o[0] = fx;
                o[1] = fy;
            }
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * _ext.dcn_v2_forward — DCNv2/src/cuda/dcn_v2_cuda.cu:42-172 with
 * modulated_deformable_im2col_gpu_kernel (dcn_v2_im2col_cuda.cu:125-195) and
 * dmcn_im2col_bilinear (:25-54).
 *
 *   out[b,o,p] = bias[o] + sum_{c,i,j} W[o,c,i,j] * columns[b, (c*kh+i)*kw+j, p]      (:123-163)
 *   columns    = mask[b, g*kh*kw + i*kw + j, p] * bilinear(x[b,c], h_im, w_im)         (:190)
 *   h_im = ho*sh - ph + i*dh + offset[b, g*2*kh*kw + 2*(i*kw+j)    , p]               (:172-178)
 *   w_im = wo*sw - pw + j*dw + offset[b, g*2*kh*kw + 2*(i*kw+j) + 1, p]
 *   value is 0 unless h_im > -1 && w_im > -1 && h_im < H && w_im < W                   (:180)
 *   g = c / (C / dg)                                                                    (:151)
 *
 * The columns value is formed in float exactly as the kernel does (same operation order);
 * the contraction is accumulated in double (acc64 != 0) or float in (c,i,j) order (acc64 == 0).
 * ------------------------------------------------------------------------------------------ */
static float bilinear_ref(const float *im, int data_width, int height, int width, float h, float w)
{
    int h_low = (int)floorf(h), w_low = (int)floorf(w);
    int h_high = h_low + 1, w_high = w_low + 1;
    float lh = h - h_low, lw = w - w_low;
    float hh = 1 - lh, hw = 1 - lw;
    float v1 = 0, v2 = 0, v3 = 0, v4 = 0;
    if (h_low >= 0 && w_low >= 0) v1 = im[h_low * data_width + w_low];
    if (h_low >= 0 && w_high <= width - 1) v2 = im[h_low * data_width + w_high];
    if (h_high <= height - 1 && w_low >= 0) v3 = im[h_high * data_width + w_low];
    if (h_high <= height - 1 && w_high <= width - 1) v4 = im[h_high * data_width + w_high];
    float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
    return (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
}

int oracle_dcn_v2_forward(const float *x, const float *weight, const float *bias,
                          const float *offset, const float *mask, float *out,
                          int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw,
                          int ph, int pw, int dh, int dw, int dg, int acc64)
{
    if (dg <= 0 || C % dg) return 1;
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
    const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    const int K = C * kh * kw, cpg = C / dg;
    const long P = (long)Ho * Wo;
#pragma omp parallel
    {
        float *col = (float *)malloc(sizeof(float) * K);
#pragma omp for collapse(2) schedule(static)
        for (int b = 0; b < B; ++b)
            for (long p = 0; p < P; ++p) {
                const int ho = (int)(p / Wo), wo = (int)(p % Wo);
                const int h_in = ho * sh - ph, w_in = wo * sw - pw;
                for (int c = 0; c < C; ++c) {
                    const int g = c / cpg;
                    const float *im = x + ((long)b * C + c) * H * W;
                    const float *offp = offset + ((long)b * dg + g) * 2 * kh * kw * P;
                    const float *mp = mask + ((long)b * dg + g) * kh * kw * P;
                    for (int i = 0; i < kh; ++i)
                        for (int j = 0; j < kw; ++j) {
                            const float oh = offp[(long)(2 * (i * kw + j)) * P + p];
                            const float ow = offp[(long)(2 * (i * kw + j) + 1) * P + p];
                            const float m = mp[(long)(i * kw + j) * P + p];
                            const float h_im = h_in + i * dh + oh;
                            const float w_im = w_in + j * dw + ow;
                            float v = 0.f;
                            if (h_im > -1 && w_im > -1 && h_im < H && w_im < W)
                                v = bilinear_ref(im, W, H, W, h_im, w_im);
                            col[(c * kh + i) * kw + j] = v * m;
                        }
                }
                for (int o = 0; o < Cout; ++o) {
                    const float *wrow = weight + (long)o * K;
                    float r;
                    if (acc64) {
                        double acc = 0.0;
                        for (int k = 0; k < K; ++k) acc += (double)wrow[k] * (double)col[k];
                        r = (float)(acc + (double)(bias ? bias[o] : 0.f));
                    } else {
                        float acc = bias ? bias[o] : 0.f;
                        for (int k = 0; k < K; ++k) acc += wrow[k] * col[k];
                        r = acc;
                    }
                    out[((long)b * Cout + o) * P + p] = r;
                }
            }
        free(col);
    }
    return 0;
}

/* per-pixel channel L2 normalise — corres_generation_arch.py:56-58, F.normalize(dim=0, eps=1e-12):
 * x[:,p] / max(||x[:,p]||_2, 1e-12) */
int oracle_channel_l2norm(const float *x, float *y, int C, long HW)
{
#pragma omp parallel for schedule(static)
    for (long p = 0; p < HW; ++p) {
        double ss = 0.0;
        for (int c = 0; c < C; ++c) ss += (double)x[(long)c * HW + p] * x[(long)c * HW + p];
        float n = (float)sqrt(ss);
        if (n < 1e-12f) n = 1e-12f;
        for (int c = 0; c < C; ++c) y[(long)c * HW + p] = x[(long)c * HW + p] / n;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * _ext.dcn_v2_backward — DCNv2/src/cuda/dcn_v2_cuda.cu:206-335 with the col2im / col2im_coord
 * kernels (dcn_v2_im2col_cuda.cu:56-123 weights, :197-254 grad_input, :256-327 grad_offset/mask).
 *
 *   gcol[b,ck,p]   = sum_o W[o,ck] * gout[b,o,p]                                        (:265-268)
 *   grad_mask      = sum_{c in g} gcol * bilinear(x[b,c], pos)       (0 outside (-1,H)x(-1,W), :300-307)
 *   grad_offset_h/w= sum_{c in g} gcol * mask * d bilinear / d h|w   (dmcn_get_coordinate_weight, :83-123)
 *   grad_input    += gcol * mask * bilinear corner weight, in-bounds corners only      (:233-252, :56-80)
 *   grad_weight[o,ck] = sum_{b,p} gout[b,o,p] * columns[b,ck,p];  grad_bias[o] = sum_{b,p} gout   (:296-330)
 * All accumulations in double.
 * ------------------------------------------------------------------------------------------ */
int oracle_dcn_v2_backward(const float *x, const float *weight, const float *offset, const float *mask,
                           const float *gout, float *gx, float *goff, float *gmask, float *gw, float *gb,
                           int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw,
                           int ph, int pw, int dh, int dw, int dg)
{
    if (dg <= 0 || C % dg) return 1;
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
    const int Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    const int T = kh * kw, K = C * T, cpg = C / dg;
    const long P = (long)Ho * Wo;
    double *dgx = (double *)calloc((size_t)B * C * H * W, sizeof(double));
    double *dgw = (double *)calloc((size_t)Cout * K, sizeof(double));
    double *dgb = (double *)calloc((size_t)Cout, sizeof(double));
    if (!dgx || !dgw || !dgb) return 2;
    for (int b = 0; b < B; ++b)
        for (long p = 0; p < P; ++p) {
            const int ho = (int)(p / Wo), wo = (int)(p % Wo);
            for (int o = 0; o < Cout; ++o) dgb[o] += gout[((long)b * Cout + o) * P + p];
            for (int g = 0; g < dg; ++g)
                for (int k = 0; k < T; ++k) {
                    const int i = k / kw, j = k % kw;
                    const float oh = offset[(((long)b * dg + g) * 2 * T + 2 * k) * P + p];
                    const float ow = offset[(((long)b * dg + g) * 2 * T + 2 * k + 1) * P + p];
                    const float m = mask[(((long)b * dg + g) * T + k) * P + p];
                    const float h_im = (float)(ho * sh - ph + i * dh) + oh;
                    const float w_im = (float)(wo * sw - pw + j * dw) + ow;
                    const int valid = h_im > -1 && w_im > -1 && h_im < H && w_im < W;
                    double acc_h = 0, acc_w = 0, acc_m = 0;
                    const int hl = (int)floorf(h_im), wl = (int)floorf(w_im), hh_ = hl + 1, wh = wl + 1;
                    const double lh = (double)h_im - hl, lw = (double)w_im - wl;
                    for (int cl = 0; cl < cpg; ++cl) {
                        const int c = g * cpg + cl, ck = c * T + k;
                        double gc = 0;
                        for (int o = 0; o < Cout; ++o) gc += (double)weight[(long)o * K + ck] * gout[((long)b * Cout + o) * P + p];
                        const float *im = x + ((long)b * C + c) * H * W;
                        double v1 = 0, v2 = 0, v3 = 0, v4 = 0;
                        if (valid) {
                            if (hl >= 0 && wl >= 0) v1 = im[hl * W + wl];
                            if (hl >= 0 && wh <= W - 1) v2 = im[hl * W + wh];
                            if (hh_ <= H - 1 && wl >= 0) v3 = im[hh_ * W + wl];
                            if (hh_ <= H - 1 && wh <= W - 1) v4 = im[hh_ * W + wh];
                        }
                        const double val = (1 - lh) * (1 - lw) * v1 + (1 - lh) * lw * v2 + lh * (1 - lw) * v3 + lh * lw * v4;
                        /* columns entry for grad_weight */
                        const double col = valid ? val * m : 0.0;
                        for (int o = 0; o < Cout; ++o) dgw[(long)o * K + ck] += (double)gout[((long)b * Cout + o) * P + p] * col;
                        if (valid) {
                            acc_m += gc * val;
                            /* d/dh: -(1-lw) v1 - lw v2 + (1-lw) v3 + lw v4 ; d/dw: -(1-lh) v1 + (1-lh) v2 - lh v3 + lh v4 */
                            acc_h += gc * m * (-(1 - lw) * v1 - lw * v2 + (1 - lw) * v3 + lw * v4);
                            acc_w += gc * m * (-(1 - lh) * v1 + (1 - lh) * v2 - lh * v3 + lh * v4);
                            const double tg = gc * m;
                            double *gim = dgx + ((long)b * C + c) * H * W;
                            if (hl >= 0 && wl >= 0) gim[hl * W + wl] += tg * (1 - lh) * (1 - lw);
                            if (hl >= 0 && wh <= W - 1) gim[hl * W + wh] += tg * (1 - lh) * lw;
                            if (hh_ <= H - 1 && wl >= 0) gim[hh_ * W + wl] += tg * lh * (1 - lw);
                            if (hh_ <= H - 1 && wh <= W - 1) gim[hh_ * W + wh] += tg * lh * lw;
                        }
                    }
                    goff[(((long)b * dg + g) * 2 * T + 2 * k) * P + p] = (float)acc_h;
                    goff[(((long)b * dg + g) * 2 * T + 2 * k + 1) * P + p] = (float)acc_w;
                    gmask[(((long)b * dg + g) * T + k) * P + p] = (float)acc_m;
                }
        }
    for (long i = 0; i < (long)B * C * H * W; ++i) gx[i] = (float)dgx[i];
    for (long i = 0; i < (long)Cout * K; ++i) gw[i] = (float)dgw[i];
    for (int o = 0; o < Cout; ++o) gb[o] = (float)dgb[o];
    free(dgx); free(dgw); free(dgb);
    return 0;
}
