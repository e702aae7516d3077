/* TEST INFRASTRUCTURE — scalar C restatement of the epipolar fusion path.  NOT product code.
 *
 * Follows SURVEY.md appendix A, which restates /root/reference/modeling/layers/epipolar.py
 * (:323-418 geometry, :199/:210 grid_sample, :295-307 similarity+softmax, :237-243 argmax +
 * weighted sum) and /root/reference/vision/multiview.py (:25-57 normalize/de_normalize,
 * :154-163 pix2coord/coord2pix).  Pinned against golden vectors produced by the reference
 * itself (tests/golden, tests/test_oracle_golden.py).
 *
 * Used only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg, for shapes
 * the numpy oracle would take minutes on.  Geometry is the infinite-homography form
 * (same epipolar line as the reference's pinv form; see oracle/epipolar_oracle.py) in
 * double precision unless geom_fp32 is set; sampling arithmetic is float like ATen's.
 *
 * Build: gcc -O2 -fopenmp -shared -fPIC -o oracle/libepi_oracle.so oracle/epi_oracle.c -lm
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define EPS_ 1e-3
#define FAR_ 10000.0
#define MASKED_ (-1e10f)

static void inv3(const double *a, double *o) {
    double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
    double det = a[0] * c00 + a[1] * c01 + a[2] * c02, id = 1.0 / det;
    o[0] = c00 * id; o[1] = (a[2] * a[7] - a[1] * a[8]) * id; o[2] = (a[1] * a[5] - a[2] * a[4]) * id;
    o[3] = c01 * id; o[4] = (a[0] * a[8] - a[2] * a[6]) * id; o[5] = (a[2] * a[3] - a[0] * a[5]) * id;
    o[6] = c02 * id; o[7] = (a[1] * a[6] - a[0] * a[7]) * id; o[8] = (a[0] * a[4] - a[1] * a[3]) * id;
}

/* per-pair constants: M = A2 A1^-1 (3x3), e2 = A2 (-A1^-1 t1) + t2, normalised by e2[2] */
static void pair_constants(const double *P1, const double *P2, double *M, double *e2) {
    double A1[9], A2[9], A1i[9], c[3];
    for (int r = 0; r < 3; r++) for (int q = 0; q < 3; q++) { A1[r * 3 + q] = P1[r * 4 + q]; A2[r * 3 + q] = P2[r * 4 + q]; }
    inv3(A1, A1i);
    for (int r = 0; r < 3; r++) c[r] = -(A1i[r * 3] * P1[3] + A1i[r * 3 + 1] * P1[7] + A1i[r * 3 + 2] * P1[11]);
    for (int r = 0; r < 3; r++) {
        e2[r] = A2[r * 3] * c[0] + A2[r * 3 + 1] * c[1] + A2[r * 3 + 2] * c[2] + P2[r * 4 + 3];
        for (int q = 0; q < 3; q++)
            M[r * 3 + q] = A2[r * 3] * A1i[q] + A2[r * 3 + 1] * A1i[3 + q] + A2[r * 3 + 2] * A1i[6 + q];
    }
    double z = e2[2]; e2[0] /= z; e2[1] /= z; e2[2] = 1.0;
}

static double sd(double v, double c) { double a = fabs(v) > c ? fabs(v) : c; return v > 0 ? a : (v < 0 ? -a : 0.0 * a); }
static float sdf(float v, float c) { float a = fabsf(v) > c ? fabsf(v) : c; return v > 0 ? a : (v < 0 ? -a : 0.0f * a); }

/* line clipping (epipolar.py:369-405): endpoints S,E in image coordinates; `c` clamps the denominators (EPS_, or 0 for the
   homogeneous line of a ray parallel to the source image plane, see line_d) */
static void clip_d(const double *l, double c, double xmin, double xmax, double ymin, double ymax, double *S, double *E) {
    double by1 = -(xmin * l[0] + l[2]) / sd(l[1], c), by2 = -(xmax * l[0] + l[2]) / sd(l[1], c);
    double bx0 = -(ymin * l[1] + l[2]) / sd(l[0], c), bx3 = -(ymax * l[1] + l[2]) / sd(l[0], c);
    double cx[4] = {bx0, xmin, xmax, bx3}, cy[4] = {ymin, by1, by2, ymax};
    int ok[4] = {bx0 >= xmin + EPS_ && bx0 < xmax - EPS_, by1 > ymin + EPS_ && by1 <= ymax - EPS_,
                 by2 >= ymin + EPS_ && by2 < ymax - EPS_, bx3 > xmin + EPS_ && bx3 <= xmax - EPS_};
    int n = 0; double px[2], py[2];
    for (int i = 0; i < 4 && n < 2; i++) if (ok[i]) { px[n] = cx[i]; py[n] = cy[i]; n++; }
    if (ok[0] + ok[1] + ok[2] + ok[3] < 2) { S[0] = E[0] = xmin - FAR_; S[1] = E[1] = ymin - FAR_; }
    else { S[0] = px[0]; S[1] = py[0]; E[0] = px[1]; E[1] = py[1]; }
}
static void clip_f(const float *l, float c, float xmin, float xmax, float ymin, float ymax, float *S, float *E) {
    const float e = (float)EPS_;
    float by1 = -(xmin * l[0] + l[2]) / sdf(l[1], c), by2 = -(xmax * l[0] + l[2]) / sdf(l[1], c);
    float bx0 = -(ymin * l[1] + l[2]) / sdf(l[0], c), bx3 = -(ymax * l[1] + l[2]) / sdf(l[0], c);
    float cx[4] = {bx0, xmin, xmax, bx3}, cy[4] = {ymin, by1, by2, ymax};
    int ok[4] = {bx0 >= xmin + e && bx0 < xmax - e, by1 > ymin + e && by1 <= ymax - e,
                 by2 >= ymin + e && by2 < ymax - e, bx3 > xmin + e && bx3 <= xmax - e};
    int n = 0; float px[2], py[2];
    for (int i = 0; i < 4 && n < 2; i++) if (ok[i]) { px[n] = cx[i]; py[n] = cy[i]; n++; }
    if (ok[0] + ok[1] + ok[2] + ok[3] < 2) { S[0] = E[0] = xmin - (float)FAR_; S[1] = E[1] = ymin - (float)FAR_; }
    else { S[0] = px[0]; S[1] = py[0]; E[0] = px[1]; E[1] = py[1]; }
}

/* l = e2 × x2 of the point x2 = M p (e2[2] == 1), returns the denominators' clamp: e2 × (x2 / x2[2]) with EPS_, or, where that
   quotient is not finite (x2[2] == 0: the ray of p is parallel to the source image plane), e2 × x2 of the homogeneous point,
   the zz -> 0 limit of the quotient form up to a factor 1/zz that grows without bound, so that the clamp never acts (0). */
static double line_d(const double *e2, const double *x2, double *l) {
    double x = x2[0] / x2[2], y = x2[1] / x2[2];
    l[0] = e2[1] - y; l[1] = x - e2[0]; l[2] = e2[0] * y - e2[1] * x;
    if (isfinite(l[0]) && isfinite(l[1]) && isfinite(l[2])) return EPS_;
    l[0] = e2[1] * x2[2] - x2[1]; l[1] = x2[0] - e2[0] * x2[2]; l[2] = e2[0] * x2[1] - e2[1] * x2[0];
    return 0.0;
}
static float line_f(const float *e2, const float *x2, float *l) {
    float x = x2[0] / x2[2], y = x2[1] / x2[2];
    l[0] = e2[1] - y; l[1] = x - e2[0]; l[2] = e2[0] * y - e2[1] * x;
    if (isfinite(l[0]) && isfinite(l[1]) && isfinite(l[2])) return (float)EPS_;
    l[0] = e2[1] * x2[2] - x2[1]; l[1] = x2[0] - e2[0] * x2[2]; l[2] = e2[0] * x2[1] - e2[1] * x2[0];
    return 0.0f;
}

int epi_oracle_forward(const float *feat_ref, const float *feat_src, const double *P_ref, const double *P_src,
                       const float *locs_in, int N, int C, int H, int W, int K, double downsample,
                       double img_scale, double softmax_scale, int correct_normalize, int align_corners,
                       int geom_fp32, float *out, float *attn, float *corr_pos, float *locs_out, int threads) {
    if (N <= 0 || C <= 0 || H < 2 || W < 2 || K < 2) return -1;
    const size_t HW = (size_t)H * W;
    const double ds = downsample, r = img_scale;
    /* fp32 pixel axes like the reference (epipolar.py:35-38 builds them from float arange) */
    const float xminf = (0.0f * (float)ds + (float)(ds / 2.0) - 0.5f) * (float)r, yminf = xminf;
    const float xmaxf = ((float)(W - 1) * (float)ds + (float)(ds / 2.0) - 0.5f) * (float)r;
    const float ymaxf = ((float)(H - 1) * (float)ds + (float)(ds / 2.0) - 0.5f) * (float)r;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    for (int n = 0; n < N; n++) {
        double M[9], e2[3];
        pair_constants(P_ref + 12 * n, P_src + 12 * n, M, e2);
        float Mf[9], e2f[3];
        for (int i = 0; i < 9; i++) Mf[i] = (float)M[i];
        for (int i = 0; i < 3; i++) e2f[i] = (float)e2[i];
        const float *fr = feat_ref + (size_t)n * C * HW, *fs = feat_src + (size_t)n * C * HW;
#pragma omp parallel
        {
            float *samp = (float *)malloc(sizeof(float) * (size_t)K * C);
            float *sim = (float *)malloc(sizeof(float) * K);
            float *gxs = (float *)malloc(sizeof(float) * 2 * K);
#pragma omp for schedule(dynamic, 16)
            for (long p = 0; p < (long)HW; p++) {
                int j = (int)(p / W), i = (int)(p % W);
                /* ---- sample locations (normalised grid coords, float like .float() at :183) ---- */
                if (locs_in) {
                    for (int k = 0; k < K; k++) {
                        const float *g = locs_in + ((((size_t)k * N + n) * H + j) * W + i) * 2;
                        gxs[2 * k] = g[0]; gxs[2 * k + 1] = g[1];
                    }
                } else {
                    float pxf = ((float)i * (float)ds + (float)(ds / 2.0) - 0.5f) * (float)r;
                    float pyf = ((float)j * (float)ds + (float)(ds / 2.0) - 0.5f) * (float)r;
                    double S[2], E[2];
                    if (geom_fp32) {
                        float x2[3], l[3], Sf[2], Ef[2];
                        for (int q = 0; q < 3; q++) x2[q] = Mf[q * 3] * pxf + Mf[q * 3 + 1] * pyf + Mf[q * 3 + 2];
                        float c = line_f(e2f, x2, l);
                        clip_f(l, c, xminf, xmaxf, yminf, ymaxf, Sf, Ef);
                        S[0] = Sf[0]; S[1] = Sf[1]; E[0] = Ef[0]; E[1] = Ef[1];
                    } else {
                        double x2[3], l[3];
                        for (int q = 0; q < 3; q++) x2[q] = M[q * 3] * pxf + M[q * 3 + 1] * pyf + M[q * 3 + 2];
                        double c = line_d(e2, x2, l);
                        clip_d(l, c, xminf, xmaxf, yminf, ymaxf, S, E);
                    }
                    for (int k = 0; k < K; k++) {
                        double t = (double)k / (double)(K - 1);
                        double g[2];
                        for (int a = 0; a < 2; a++) {
                            double v, pix; int size = a == 0 ? W : H;
                            if (geom_fp32) { float vf = (float)S[a] + ((float)E[a] - (float)S[a]) * (float)t;
                                float pf = (vf / (float)r + 0.5f - (float)(ds / 2.0)) / (float)ds;
                                g[a] = correct_normalize ? -1.0f + 2.0f * pf / (float)(size - 1) : -1.0f + 2.0f * (pf + 0.5f) / (float)size;
                            } else { v = S[a] + (E[a] - S[a]) * t; pix = (v / r + 0.5 - ds / 2.0) / ds;
                                g[a] = correct_normalize ? -1.0 + 2.0 * pix / (size - 1) : -1.0 + 2.0 * (pix + 0.5) / size; }
                        }
                        gxs[2 * k] = (float)g[0]; gxs[2 * k + 1] = (float)g[1];
                    }
                }
                if (locs_out)
                    for (int k = 0; k < K; k++) {
                        float *g = locs_out + ((((size_t)k * N + n) * H + j) * W + i) * 2;
                        g[0] = gxs[2 * k]; g[1] = gxs[2 * k + 1];
                    }
                /* ---- K bilinear samples, zero padding (epipolar.py:199) ---- */
                for (int k = 0; k < K; k++) {
                    float gx = gxs[2 * k], gy = gxs[2 * k + 1], ix, iy;
                    if (align_corners) { ix = (gx + 1.f) / 2.f * (float)(W - 1); iy = (gy + 1.f) / 2.f * (float)(H - 1); }
                    else { ix = ((gx + 1.f) * (float)W - 1.f) / 2.f; iy = ((gy + 1.f) * (float)H - 1.f) / 2.f; }
                    float x0 = floorf(ix), y0 = floorf(iy), x1 = x0 + 1.f, y1 = y0 + 1.f;
                    float w[4] = {(x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)};
                    float tx[4] = {x0, x1, x0, x1}, ty[4] = {y0, y0, y1, y1};
                    float *s = samp + (size_t)k * C;
                    memset(s, 0, sizeof(float) * C);
                    for (int t = 0; t < 4; t++) {
                        if (!(tx[t] >= 0.f && tx[t] <= (float)(W - 1) && ty[t] >= 0.f && ty[t] <= (float)(H - 1))) continue;
                        const float *src = fs + (size_t)ty[t] * W + (size_t)tx[t];
                        for (int c = 0; c < C; c++) s[c] += w[t] * src[(size_t)c * HW];
                    }
                    double acc = 0.0;      /* the sum order of ATen is unspecified; double keeps the oracle order-free */
                    for (int c = 0; c < C; c++) acc += (double)(s[c] * fr[(size_t)c * HW + p]);
                    float v = (float)acc;
                    if (v == 0.0f) v = MASKED_;          /* :298 */
                    sim[k] = v * (float)softmax_scale;   /* :306 */
                }
                /* ---- softmax over K (:307), argmax (:237), weighted sum (:243) ---- */
                float mx = sim[0];
                for (int k = 1; k < K; k++) if (sim[k] > mx) mx = sim[k];
                double sum = 0.0;
                for (int k = 0; k < K; k++) { sim[k] = expf(sim[k] - mx); sum += sim[k]; }
                int best = 0;
                for (int k = 0; k < K; k++) { sim[k] = (float)(sim[k] / sum); if (sim[k] > sim[best]) best = k; }
                if (attn) for (int k = 0; k < K; k++) attn[((size_t)n * K + k) * HW + p] = sim[k];
                if (corr_pos) {
                    float gx = gxs[2 * best], gy = gxs[2 * best + 1];
                    float *cp = corr_pos + ((size_t)n * HW + p) * 2;
                    if (correct_normalize) { cp[0] = (gx + 1.f) * (float)(W - 1) / 2.f; cp[1] = (gy + 1.f) * (float)(H - 1) / 2.f; }
                    else { cp[0] = (gx + 1.f) * (float)W / 2.f - .5f; cp[1] = (gy + 1.f) * (float)H / 2.f - .5f; }
                }
                for (int c = 0; c < C; c++) {
                    double acc = 0.0;
                    for (int k = 0; k < K; k++) acc += (double)(samp[(size_t)k * C + c] * sim[k]);
                    out[((size_t)n * C + c) * HW + p] = (float)acc;
                }
            }
            free(samp); free(sim); free(gxs);
        }
    }
    return 0;
}
