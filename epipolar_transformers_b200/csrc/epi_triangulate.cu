// epi_triangulate.cu — linear (DLT) triangulation of every (frame, joint) of a multi-view batch in one launch, one thread per
// problem, as pymvg's find3d computes it after the confidence-based view selection of the reference's 'pymvg' mode:
//   1. views: t = conf_thres (fp64); sel = {v : score[v] > (float)t}; stop if t < −1; if |sel| <= 1, t −= 0.05 and repeat
//   2. A: per selected view, in increasing view order, the rows x·M[2] − M[0] and y·M[2] − M[1] (fp64)
//   3. X = v[:3] / v[3], v the right singular vector of A's smallest singular value
// A is never stored: each row is folded into a 4x4 upper-triangular R by Givens rotations as it is formed (A = QR, so A and R
// have the same right singular vectors), and R's SVD is taken by one-sided Jacobi.  AᵀA is never formed: its condition number
// is the square of A's, and a camera's translation column (mm times the focal length, ~1e6) against its rotation columns
// (~1e3) would leave too few of fp64's digits for the null vector.
#include "epi_kernels.cuh"

#include <cfloat>

namespace epi {

// R <- the R of [R; a] (a: one row of A), by the Givens rotations that zero a left to right.  A NaN in a spreads to R.
__host__ __device__ __forceinline__ void givens_fold_row(double (&R)[4][4], double (&a)[4]) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
        if (a[i] != 0.0) {
            const double r = hypot(R[i][i], a[i]);
            const double c = R[i][i] / r, s = a[i] / r;
            R[i][i] = r;
#pragma unroll
            for (int k = i + 1; k < 4; k++) {
                const double rk = R[i][k], ak = a[k];
                R[i][k] = c * rk + s * ak;
                a[k] = c * ak - s * rk;
            }
        }
    }
}

// The right singular vector of R's smallest singular value, by one-sided (Hestenes) Jacobi: rotate pairs of R's columns until
// they are orthogonal to working precision; the accumulated rotations are V, and the column norms the singular values.
__host__ __device__ __forceinline__ void jacobi_null_vector(double (&R)[4][4], double (&v)[4]) {
    double Vm[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) Vm[i][k] = i == k ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; sweep++) {
        bool rotated = false;
#pragma unroll
        for (int p = 0; p < 3; p++) {
#pragma unroll
            for (int q = p + 1; q < 4; q++) {
                double alpha = 0.0, beta = 0.0, gamma = 0.0;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    alpha += R[i][p] * R[i][p];
                    beta += R[i][q] * R[i][q];
                    gamma += R[i][p] * R[i][q];
                }
                if (fabs(gamma) > DBL_EPSILON * sqrt(alpha) * sqrt(beta)) {      // false for a NaN gamma: the sweep ends
                    rotated = true;
                    const double zeta = (beta - alpha) / (2.0 * gamma);
                    const double t = copysign(1.0, zeta) / (fabs(zeta) + hypot(1.0, zeta));
                    const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const double rp = R[i][p], rq = R[i][q];
                        R[i][p] = c * rp - s * rq;
                        R[i][q] = s * rp + c * rq;
                        const double vp = Vm[i][p], vq = Vm[i][q];
                        Vm[i][p] = c * vp - s * vq;
                        Vm[i][q] = s * vp + c * vq;
                    }
                }
            }
        }
        if (!rotated) break;
    }
    double best = INFINITY;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double n2 = R[0][k] * R[0][k] + R[1][k] * R[1][k] + R[2][k] * R[2][k] + R[3][k] * R[3][k];
        if (k == 0 || n2 < best) {
            best = n2;
#pragma unroll
            for (int i = 0; i < 4; i++) v[i] = Vm[i][k];
        }
    }
}

// locs [V,N,J,2], scores [V,N,J], P [V,N,3,4] -> X [N,J,3], n_used [N,J]; thread = n·J + j
template <typename PT>
__global__ void __launch_bounds__(128) epi_triangulate_kernel(const float *__restrict__ locs, const float *__restrict__ scores,
                                                              const PT *__restrict__ P, double conf_thres, int V, int N, int J,
                                                              double *__restrict__ X, int *__restrict__ n_used) {
    const int NJ = N * J;
    const long long p64 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p64 >= NJ) return;
    const int p = (int)p64, n = p / J;
    // ---- 1. the views: a float32 compare against (float)t, t stepped in fp64 as the reference's Python float ----
    float smax = -INFINITY;                              // no score above it: a pass at (float)t >= smax selects nothing
    for (int v = 0; v < V; v++) smax = fmaxf(smax, __ldg(scores + (size_t)v * NJ + p));      // fmaxf skips NaN
    double t = conf_thres;
    unsigned long long sel;
    for (;;) {
        const float tf = (float)t;
        sel = 0ull;
        if (smax > tf)
            for (int v = 0; v < V; v++)
                if (__ldg(scores + (size_t)v * NJ + p) > tf) sel |= 1ull << v;
        if (t < -1.0) break;
        if (__popcll(sel) <= 1) { t -= 0.05; continue; }
        break;
    }
    const int used = __popcll(sel);
    // ---- 2. A's rows, folded into R as they are formed ----
    double R[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) R[i][k] = 0.0;
    bool finite = true;
    for (unsigned long long s = sel; s; s &= s - 1) {
        const int v = __ffsll((long long)s) - 1;
        const PT *M = P + ((size_t)v * N + n) * 12;
        double m[12];
#pragma unroll
        for (int i = 0; i < 12; i++) { m[i] = (double)M[i]; finite &= isfinite(m[i]); }
        const float2 xy = __ldg(reinterpret_cast<const float2 *>(locs) + (size_t)v * NJ + p);
        const double x = xy.x, y = xy.y;
        finite &= isfinite(x) && isfinite(y);
        double a[4], b[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            a[k] = x * m[8 + k] - m[k];
            b[k] = y * m[8 + k] - m[4 + k];
        }
        givens_fold_row(R, a);
        givens_fold_row(R, b);
    }
    // ---- 3. the null vector and the division ----
    double Xp[3] = {NAN, NAN, NAN};
    if (used >= 2 && finite) {
        double v[4];
        jacobi_null_vector(R, v);
        Xp[0] = v[0] / v[3]; Xp[1] = v[1] / v[3]; Xp[2] = v[2] / v[3];
    }
    X[3 * (size_t)p] = Xp[0];
    X[3 * (size_t)p + 1] = Xp[1];
    X[3 * (size_t)p + 2] = Xp[2];
    n_used[p] = used;
}

cudaError_t launch_triangulate(const float *locs, const float *scores, const void *P, bool P_f64, double conf_thres, int V, int N,
                               int J, double *X, int *n_used, cudaStream_t st) {
    const int NJ = N * J, blocks = (int)(((long long)NJ + 127) / 128);
    if (P_f64)
        epi_triangulate_kernel<double><<<blocks, 128, 0, st>>>(locs, scores, static_cast<const double *>(P), conf_thres, V, N, J, X, n_used);
    else
        epi_triangulate_kernel<float><<<blocks, 128, 0, st>>>(locs, scores, static_cast<const float *>(P), conf_thres, V, N, J, X, n_used);
    return cudaGetLastError();
}

}  // namespace epi
