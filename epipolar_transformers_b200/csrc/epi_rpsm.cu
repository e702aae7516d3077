// epi_rpsm.cu — the reference's recursive pictorial-structure model (KEYPOINT.TRIANGULATION = 'rpsm') for a batch of frames:
// the 3-D pose on a cube of bins around a root point, refined on ever smaller cubes around each joint, with no host sync.
//
// Every float32 operation is one IEEE op in a fixed order (explicit __f*_rn intrinsics: nvcc would contract a*b+c), so
// oracle/rpsm_oracle.py restates the arithmetic bit for bit.  The points the reference fixes:
//  1. Grid.  g = torch.linspace(-s/2, s/2, n) in float32: start = fl(-s/2), end = fl(s/2), step = fl((end - start)/(n - 1));
//     g[i] = fma(step, i, start) for i < n/2, else fma(-step, n-1-i, end) (the CPU kernel's two halves, each one fused
//     multiply-add).  Coordinate = fl(g[i] + fl(c)); bin b = (ix·n + iy)·n + iz (meshgrid 'ij').  Level 0: size GRID_SIZE,
//     n = FIRST_NBINS, one grid for all joints around the caller's root point.  Recursion r = 1..RECUR_DEPTH: n = RECUR_NBINS
//     per axis around each joint's current estimate (which is not itself a bin), size GRID_SIZE / FIRST_NBINS / RECUR_NBINS^(r-1)
//     divided in fp64.  The host computes the 1-D grids (g0, gr) with std::fma, so the device only adds the centre.
//  2. Unary.  Per view v, q = P_v·[X,1] as ((P0·x + P1·y) + P2·z) + P3 per row; (u, t) = (q0/q2, q1/q2); (a, b) = T_v·[u, t, 1]
//     as (T0·u + T1·t) + T2; a' = (a·w)/IMAGE_SIZE[0], b' = (b·h)/IMAGE_SIZE[1]; grid = ((a'/(h-1))·2 - 1, (b'/(w-1))·2 - 1)
//     (the reference's h/w swap).  Then make_taps (epi_common.cuh: grid2pix, floor, the four weights) and the sum of the
//     in-bounds taps' w·value, nw, ne, sw, se, from 0 (zero padding; a tap in bounds counts even at weight 0).  The joint's
//     unary is s_0 + s_1 + ... in view order.  A bin outside every view has a unary of exactly 0.
//  3. Pairwise.  Level 0: the caller's packed 0/1 mask per edge.  Recursions: d = fl(fl(X_p - X_c) + 1e-6) per axis (torch's
//     pairwise_distance eps inside the norm), n2 = fma(d2, d2, fma(d1, d1, d0·d0)), dist = fl(sqrt(n2) + 1e-9f),
//     on = |fl(dist - L)| < tol, L the float32 limb length, tol the float32 tolerance.
//  4. Max-product, children before parents: m[p] = max_k pw[p,k]·E_c[k], s[p] = its arg-max; E_parent = ((U·m_c1)·m_c2)·...
//     in ascending child order.  torch.max's semantics: the first NaN wins; otherwise the largest value, the lowest index
//     among equals (+0 == -0).  A masked-off entry is 0·E_c[k]: ±0, or NaN when E_c[k] is not finite.
//  5. Decode.  The root's bin is the first arg-max of its energy (np.argmax); each child's is read from s top-down; the pose
//     is the bins' coordinates, and the next recursion is centred on it.
//
// Launches: unary0 (one thread per (frame, bin), every view projected once, all J maps sampled from it), one max-product
// launch per tree depth (the mask tiled through shared memory against 32 frames' child energies; one lane per frame, so
// the mask word and the bit loop are warp-uniform), and one CTA per frame for the root arg-max, the back-tracking and
// every recursion, in shared memory.
#include "epi_kernels.cuh"

namespace epi {

namespace {

constexpr int kMpRows = 64;          // parent bins per max-product CTA (8 per warp)
constexpr int kMpRowsPerWarp = 8;
constexpr int kMpChunk = 512;        // child bins staged per step
constexpr int kMpWords = kMpChunk / 32;
constexpr size_t kMpSmem = sizeof(float) * 32 * (kMpChunk + 1) + sizeof(uint2) * kMpWords * 32;
constexpr int kFinalThreads = 256;
constexpr int kMaxRB = kRpsmMaxNbinsR * kRpsmMaxNbinsR * kRpsmMaxNbinsR;

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fffffff); }

// (v, i) before (bv, bi) in a first-NaN / first-maximum arg-max (torch.max, np.argmax); i < 0 is "none"
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
    if (i < 0) return false;
    if (bi < 0) return true;
    const bool vn = v != v, bn = bv != bv;
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// 2. the normalised sample location of point (x, y, z) in view v's heat-map
__device__ __forceinline__ void project(const float *__restrict__ M, const float *__restrict__ T, float x, float y, float z,
                                       const RpsmArgs &a, float &gx, float &gy) {
    float q[3];
#pragma unroll
    for (int r = 0; r < 3; r++)
        q[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(M + 4 * r), x), __fmul_rn(__ldg(M + 4 * r + 1), y)),
                                   __fmul_rn(__ldg(M + 4 * r + 2), z)), __ldg(M + 4 * r + 3));
    const float u = __fdiv_rn(q[0], q[2]), t = __fdiv_rn(q[1], q[2]);
    float ca = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(T), u), __fmul_rn(__ldg(T + 1), t)), __ldg(T + 2));
    float cb = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(T + 3), u), __fmul_rn(__ldg(T + 4), t)), __ldg(T + 5));
    ca = __fdiv_rn(__fmul_rn(ca, (float)a.w), a.img0);
    cb = __fdiv_rn(__fmul_rn(cb, (float)a.h), a.img1);
    gx = __fsub_rn(__fmul_rn(__fdiv_rn(ca, (float)(a.h - 1)), 2.f), 1.f);
    gy = __fsub_rn(__fmul_rn(__fdiv_rn(cb, (float)(a.w - 1)), 2.f), 1.f);
}

// bilinear, zero padding: the in-bounds taps' w·value summed nw, ne, sw, se from 0
__device__ __forceinline__ float sample(const float *__restrict__ map, const Taps &t, int h, int w) {
    const bool x0 = t.x0 >= 0 && t.x0 < w, x1 = t.x0 + 1 >= 0 && t.x0 + 1 < w;
    const bool y0 = t.y0 >= 0 && t.y0 < h, y1 = t.y0 + 1 >= 0 && t.y0 + 1 < h;
    const float *p = map + (ptrdiff_t)t.y0 * w + t.x0;
    float s = 0.f;
    if (x0 && y0) s = __fadd_rn(s, __fmul_rn(t.w[0], __ldg(p)));
    if (x1 && y0) s = __fadd_rn(s, __fmul_rn(t.w[1], __ldg(p + 1)));
    if (x0 && y1) s = __fadd_rn(s, __fmul_rn(t.w[2], __ldg(p + w)));
    if (x1 && y1) s = __fadd_rn(s, __fmul_rn(t.w[3], __ldg(p + w + 1)));
    return s;
}

// 3. the recursions' pairwise term
__device__ __forceinline__ float limb_ok(const float *xp, const float *xc, float L, float tol) {
    const float d0 = __fadd_rn(__fsub_rn(xp[0], xc[0]), 1e-6f), d1 = __fadd_rn(__fsub_rn(xp[1], xc[1]), 1e-6f);
    const float d2 = __fadd_rn(__fsub_rn(xp[2], xc[2]), 1e-6f);
    const float dist = __fadd_rn(__fsqrt_rn(__fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmul_rn(d0, d0)))), 1e-9f);
    return fabsf(__fsub_rn(dist, L)) < tol ? 1.f : 0.f;
}

// ---- level 0, unary: thread = (frame, bin); U[n, j, b] ----
__global__ void __launch_bounds__(128) rpsm_unary0_kernel(const __grid_constant__ RpsmArgs a, int J) {
    const int n = blockIdx.x, b = blockIdx.y * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    const int n0 = a.n0;
    const float x = __fadd_rn(a.g0[b / (n0 * n0)], __ldg(a.root + 3 * n));
    const float y = __fadd_rn(a.g0[(b / n0) % n0], __ldg(a.root + 3 * n + 1));
    const float z = __fadd_rn(a.g0[b % n0], __ldg(a.root + 3 * n + 2));
    const size_t hw = (size_t)a.h * a.w;
    float acc[kRpsmMaxJoints];
    for (int v = 0; v < a.V; v++) {
        const size_t vn = (size_t)v * a.N + n;
        float gx, gy;
        project(a.P + vn * 12, a.crop + vn * 6, x, y, z, a, gx, gy);
        const Taps t = make_taps(gx, gy, a.h, a.w, a.align);
        const float *maps = a.heat + vn * J * hw;
#pragma unroll
        for (int j = 0; j < kRpsmMaxJoints; j++) {
            if (j < J) {
                const float s = sample(maps + j * hw, t, a.h, a.w);
                acc[j] = v == 0 ? s : __fadd_rn(acc[j], s);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < kRpsmMaxJoints; j++)
        if (j < J) a.energy[((size_t)n * J + j) * a.B + b] = acc[j];
}

// ---- level 0, max-product over the edges whose parent is pars[blockIdx.z]: lane = frame, warp = 8 parent bins ----
struct Parents { int n; signed char p[kRpsmMaxJoints]; };

__global__ void __launch_bounds__(256, 2) rpsm_maxprod0_kernel(const __grid_constant__ RpsmArgs a,
                                                            const __grid_constant__ RpsmTree t, const __grid_constant__ Parents pars) {
    extern __shared__ float smem[];
    float *sE = smem;                                                             // [32 frames][kMpChunk + 1]
    uint2 *sBits = reinterpret_cast<uint2 *>(smem + 32 * (kMpChunk + 1));        // [word][frame]: (non-finite, NaN) bits
    const int parent = pars.p[blockIdx.z];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + lane, J = t.J, B = a.B, WPR = (B + 31) / 32;
    const bool live = n < a.N;
    const int row0 = blockIdx.y * kMpRows + warp * kMpRowsPerWarp;
    float acc[kMpRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kMpRowsPerWarp; r++)
        acc[r] = live && row0 + r < B ? a.energy[((size_t)n * J + parent) * B + row0 + r] : 0.f;
    for (int c = 0; c < J; c++) {
        if (t.parent[c] != parent) continue;                                      // children in ascending order
        const int e = t.edge[c];
        float best[kMpRowsPerWarp], zval[kMpRowsPerWarp];
        int idx[kMpRowsPerWarp], koff[kMpRowsPerWarp];
        bool isnan_[kMpRowsPerWarp];
#pragma unroll
        for (int r = 0; r < kMpRowsPerWarp; r++) { best[r] = 0.f; zval[r] = 0.f; idx[r] = -1; koff[r] = -1; isnan_[r] = false; }
        for (int k0 = 0; k0 < B; k0 += kMpChunk) {
            __syncthreads();                                                      // the previous chunk's readers are done
            for (int i = threadIdx.x; i < 32 * kMpChunk; i += blockDim.x) {
                const int f = i / kMpChunk, k = i % kMpChunk, nn = blockIdx.x * 32 + f;
                sE[f * (kMpChunk + 1) + k] = nn < a.N && k0 + k < B ? a.energy[((size_t)nn * J + c) * B + k0 + k] : 0.f;
            }
            __syncthreads();
            for (int i = warp; i < 32 * kMpWords; i += blockDim.x / 32) {
                const int f = i / kMpWords, wd = i % kMpWords;
                const float v = sE[f * (kMpChunk + 1) + wd * 32 + lane];
                const unsigned nf = __ballot_sync(0xffffffffu, !isfinite(v)), nan = __ballot_sync(0xffffffffu, v != v);
                if (lane == 0) sBits[wd * 32 + f] = make_uint2(nf, nan);
            }
            __syncthreads();
            const int nw = min(kMpWords, WPR - k0 / 32);
            const float *myE = sE + lane * (kMpChunk + 1);
#pragma unroll
            for (int r = 0; r < kMpRowsPerWarp; r++) {
                const int p = row0 + r;
                if (p >= B) break;                                                // warp-uniform
                const uint32_t *mrow = a.mask + ((size_t)e * B + p) * WPR + k0 / 32;
                const uint32_t mine = lane < nw ? __ldg(mrow + lane) : 0u;
                for (int wd = 0; wd < nw; wd++) {
                    const int kb = k0 + wd * 32;
                    const uint32_t valid = B - kb >= 32 ? 0xffffffffu : (1u << (B - kb)) - 1u;
                    const uint32_t on = __shfl_sync(0xffffffffu, mine, wd) & valid, off = ~on & valid;
                    const uint2 fb = sBits[wd * 32 + lane];
                    if (koff[r] < 0 && off) {                                     // the first masked-off bin: the ±0 candidate
                        koff[r] = kb + __ffs(off) - 1;
                        zval[r] = __fmul_rn(0.f, myE[koff[r] - k0]);
                    }
                    const uint32_t nanc = (off & fb.x) | (on & fb.y);            // entries that are NaN: 0·(±inf, NaN), 1·NaN
                    if (!isnan_[r] && nanc) { isnan_[r] = true; best[r] = qnan(); idx[r] = kb + __ffs(nanc) - 1; }
                    for (uint32_t bits = on; bits; bits &= bits - 1) {
                        const int bit = __ffs(bits) - 1;
                        const float v = myE[kb - k0 + bit];
                        if (!isnan_[r] && (idx[r] < 0 || v > best[r])) { best[r] = v; idx[r] = kb + bit; }
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kMpRowsPerWarp; r++) {
            const int p = row0 + r;
            if (p >= B) break;
            float m = best[r];
            int s = idx[r];
            if (!isnan_[r] && koff[r] >= 0 && (s < 0 || best[r] < 0.f || (best[r] == 0.f && koff[r] < s))) { m = zval[r]; s = koff[r]; }
            acc[r] = __fmul_rn(acc[r], m);
            if (live) a.state[((size_t)n * t.E + e) * B + p] = (int16_t)s;
        }
    }
#pragma unroll
    for (int r = 0; r < kMpRowsPerWarp; r++)
        if (live && row0 + r < B) a.energy[((size_t)n * J + parent) * B + row0 + r] = acc[r];
}

// block-wide first arg-max of v[0..count) (global or shared); every thread gets the index
__device__ int block_argmax(const float *v, int count, float *rv, int *ri) {
    float bv = 0.f;
    int bi = -1;
    for (int k = threadIdx.x; k < count; k += blockDim.x) {
        const float x = v[k];
        if (better(x, k, bv, bi)) { bv = x; bi = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { rv[threadIdx.x >> 5] = bv; ri[threadIdx.x >> 5] = bi; }
    __syncthreads();
    bv = rv[0];
    bi = ri[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++)
        if (better(rv[w], ri[w], bv, bi)) { bv = rv[w]; bi = ri[w]; }
    return bi;
}

// ---- the root's arg-max, the back-tracking and every recursion: one CTA per frame ----
__global__ void __launch_bounds__(kFinalThreads) rpsm_recurse_kernel(const __grid_constant__ RpsmArgs a,
                                                                           const __grid_constant__ RpsmTree t) {
    __shared__ float sX[kRpsmMaxJoints * kMaxRB * 3], sE[kRpsmMaxJoints * kMaxRB], sPose[kRpsmMaxJoints * 3];
    __shared__ signed char sS[kRpsmMaxJoints * kMaxRB];
    __shared__ int sBin[kRpsmMaxJoints];
    __shared__ float rv[kFinalThreads / 32];
    __shared__ int ri[kFinalThreads / 32];
    const int n = blockIdx.x, J = t.J, tid = threadIdx.x;
    // level 0: decode
    const int rootbin = block_argmax(a.energy + ((size_t)n * J + t.root) * a.B, a.B, rv, ri);
    if (tid == 0) {
        sBin[t.root] = rootbin;
        for (int i = 1; i < J; i++) {
            const int j = t.bfs[i];
            sBin[j] = a.state[((size_t)n * t.E + t.edge[j]) * a.B + sBin[t.parent[j]]];
        }
    }
    __syncthreads();
    if (tid < J) {
        const int b = sBin[tid], n0 = a.n0;
        sPose[3 * tid] = __fadd_rn(a.g0[b / (n0 * n0)], __ldg(a.root + 3 * n));
        sPose[3 * tid + 1] = __fadd_rn(a.g0[(b / n0) % n0], __ldg(a.root + 3 * n + 1));
        sPose[3 * tid + 2] = __fadd_rn(a.g0[b % n0], __ldg(a.root + 3 * n + 2));
    }
    const int nr = a.nr, RB = nr * nr * nr, JR = J * RB;
    const size_t hw = (size_t)a.h * a.w;
    for (int r = 0; r < a.depth; r++) {
        __syncthreads();
        // grids and unaries
        for (int it = tid; it < JR; it += blockDim.x) {
            const int j = it / RB, b = it % RB;
            const float x = __fadd_rn(a.gr[r][b / (nr * nr)], sPose[3 * j]);
            const float y = __fadd_rn(a.gr[r][(b / nr) % nr], sPose[3 * j + 1]);
            const float z = __fadd_rn(a.gr[r][b % nr], sPose[3 * j + 2]);
            sX[3 * it] = x; sX[3 * it + 1] = y; sX[3 * it + 2] = z;
            float u = 0.f;
            for (int v = 0; v < a.V; v++) {
                const size_t vn = (size_t)v * a.N + n;
                float gx, gy;
                project(a.P + vn * 12, a.crop + vn * 6, x, y, z, a, gx, gy);
                const float s = sample(a.heat + (vn * J + j) * hw, make_taps(gx, gy, a.h, a.w, a.align), a.h, a.w);
                u = v == 0 ? s : __fadd_rn(u, s);
            }
            sE[it] = u;
        }
        // max-product, deepest parents first
        for (int d = t.max_depth; d >= 1; d--) {
            __syncthreads();
            for (int it = tid; it < JR; it += blockDim.x) {
                const int pj = it / RB, pa = it % RB;
                if (t.depth[pj] != d - 1) continue;
                float Ep = sE[it];
                for (int c = 0; c < J; c++) {
                    if (t.parent[c] != pj) continue;
                    const float L = __ldg(a.limb + (size_t)n * t.E + t.edge[c]);
                    float bv = 0.f;
                    int bi = -1;
                    for (int b = 0; b < RB; b++) {
                        const float v = __fmul_rn(limb_ok(sX + 3 * it, sX + 3 * (c * RB + b), L, a.tol), sE[c * RB + b]);
                        if (better(v, b, bv, bi)) { bv = v; bi = b; }
                    }
                    sS[c * RB + pa] = (signed char)bi;
                    Ep = __fmul_rn(Ep, bv);
                }
                sE[it] = Ep;
            }
        }
        __syncthreads();
        const int rb = block_argmax(sE + t.root * RB, RB, rv, ri);
        if (tid == 0) {
            sBin[t.root] = rb;
            for (int i = 1; i < J; i++) {
                const int j = t.bfs[i];
                sBin[j] = sS[j * RB + sBin[t.parent[j]]];
            }
        }
        __syncthreads();
        if (tid < J) {
            const int k = tid * RB + sBin[tid];
            sPose[3 * tid] = sX[3 * k]; sPose[3 * tid + 1] = sX[3 * k + 1]; sPose[3 * tid + 2] = sX[3 * k + 2];
        }
    }
    __syncthreads();
    for (int i = tid; i < 3 * J; i += blockDim.x) a.pose[(size_t)n * J * 3 + i] = sPose[i];
}

// ---- the packed level-0 mask: thread = one word ----
struct G0 { float g[kRpsmMaxNbins0]; };
__global__ void __launch_bounds__(256) rpsm_pack_kernel(const float *__restrict__ dense, const float *__restrict__ limb, int E, int n0,
                                                        const __grid_constant__ G0 g0, float tol,
                                                        uint32_t *__restrict__ packed) {
    const int B = n0 * n0 * n0, WPR = (B + 31) / 32;
    const long long wid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (wid >= (long long)E * B * WPR) return;
    const int wd = (int)(wid % WPR), p = (int)((wid / WPR) % B), e = (int)(wid / ((long long)WPR * B));
    uint32_t bits = 0;
    const float xp[3] = {g0.g[p / (n0 * n0)], g0.g[(p / n0) % n0], g0.g[p % n0]};
    for (int i = 0; i < 32; i++) {
        const int k = wd * 32 + i;
        if (k >= B) break;
        bool on;
        if (dense) {
            on = __ldg(dense + ((size_t)e * B + p) * B + k) != 0.f;
        } else {
            // the grid centred at the origin: fl(g + 0) = g
            const float xc[3] = {g0.g[k / (n0 * n0)], g0.g[(k / n0) % n0], g0.g[k % n0]};
            on = limb_ok(xp, xc, __ldg(limb + e), tol) != 0.f;
        }
        bits |= (uint32_t)on << i;
    }
    packed[wid] = bits;
}

}  // namespace

cudaError_t launch_rpsm(const RpsmArgs &a, const RpsmTree &t, cudaStream_t st, int *launches) {
    int n = 0;
    rpsm_unary0_kernel<<<dim3(a.N, (a.B + 127) / 128), 128, 0, st>>>(a, t.J);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    n++;
    e = cudaFuncSetAttribute(rpsm_maxprod0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMpSmem);   // per device
    if (e != cudaSuccess) return e;
    for (int d = t.max_depth; d >= 1; d--) {
        Parents pars{};
        for (int j = 0; j < t.J; j++)
            if (t.depth[j] == d - 1) {
                bool has_child = false;
                for (int c = 0; c < t.J; c++) has_child |= t.parent[c] == j;
                if (has_child) pars.p[pars.n++] = (signed char)j;
            }
        rpsm_maxprod0_kernel<<<dim3((a.N + 31) / 32, (a.B + kMpRows - 1) / kMpRows, pars.n), 256, kMpSmem, st>>>(a, t, pars);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        n++;
    }
    rpsm_recurse_kernel<<<a.N, kFinalThreads, 0, st>>>(a, t);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    *launches = n + 1;
    return cudaSuccess;
}

cudaError_t launch_rpsm_pack(const float *dense, const float *limb, int E, int n0, const float *g0, float tol, uint32_t *packed,
                             cudaStream_t st) {
    G0 g{};
    for (int i = 0; i < n0; i++) g.g[i] = g0[i];
    const int B = n0 * n0 * n0;
    const long long words = (long long)E * B * ((B + 31) / 32);
    rpsm_pack_kernel<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(dense, limb, E, n0, g, tol, packed);
    return cudaGetLastError();
}

}  // namespace epi
