// epi_fusion_bwd.cu — backward of the fused epipolar attention (SURVEY.md 8f rank 1): one warp per reference pixel.
//
// Forward per reference pixel (epipolar.py:188-247, sample locations are constants, :178 `torch.no_grad`):
//   s_k = Σ_t w_kt·F[p_kt]   (grid_sample of the source map; "keys" = other1, "values" = other2, same numbers)
//   sim_k = q·s_k ;  masked_k = (sim_k == 0) -> -1e10 (:298, an assignment: no gradient) ;  a = softmax(scale·sim)
//   out  = Σ_k a_k·s_k
// Backward, given g = dL/dout [C] (and optionally dL/da from a loss on the returned attention):
//   dL/da_k  = g·s_k (+ dL/da_k given)          dL/dx = a ⊙ (dL/da − Σ_j a_j dL/da_j)        dsim_k = masked_k ? 0 : scale·dx_k
//   dL/dq    = Σ_k dsim_k·s_k
//   dL/dF[p] += w_kt·( [values] a_k·g  +  [keys] dsim_k·q )       for every tap (k,t) -> p      (OTHER_GRAD: epipolar.py:141-153)
// Two passes over the K samples (the second one re-gathers the taps instead of storing K·C values); the source gradient is
// accumulated with 16-byte vector atomics into a pixel-major fp32 map (zeroed by the host wrapper) and transposed to the
// caller's layout afterwards.  The attention weights saved by the forward are reused, so no softmax is recomputed.
// The deterministic backward (EpiFusionBwdParams.deterministic) runs the same kernel as a coefficient pass that stores
// (cv_k, ck_k) and a per-pair bound instead of scattering, then a fixed-point scatter with int64 atomics (DESIGN.md §3.5, §5).
// The views form (epi_fusion_views_backward_f32) launches the same kernels with a trailing BwdViews parameter: pair n then reads
// its query item and its source item of one staged map through pair_items, and the source terms of every pair that names an item
// land in that item's accumulator.  Without the parameter the pack is empty and both items are n.
#include "epi_kernels.cuh"

namespace epi {

// (query item, source item) of pair n: n itself in the one-pair form, pair_items in the views form
__device__ __forceinline__ PairItems bwd_items(int n) { return {n, n}; }
__device__ __forceinline__ PairItems bwd_items(int n, const BwdViews &vw) { return pair_items(n, vw.n_ref, vw.n_views, vw.vs); }
// fixed-point scale of source item `item`: the pair's own bound word in the one-pair form; in the views form the item's word (the
// largest bound of the pairs that scatter into it) and their number (det_item_scale)
__device__ __forceinline__ bool bwd_scale(unsigned word, int HW, int item, int &s) { return det_scale(word, HW, s); }
__device__ __forceinline__ bool bwd_scale(unsigned word, int HW, int item, int &s, const BwdViews &vw) {
    return det_item_scale(word, HW, view_source_count(item / vw.n_ref, vw.n_views, vw.vs), s);
}

namespace bwd {
constexpr int TILE_PIX = 32;
constexpr int WARPS = 8;
constexpr int MAXKCH = 8;                        // K <= 256
}  // namespace bwd

// [C][33] shared tile of the TILE_PIX pixels from p0 of one [C,H,W] item (any strides; zero beyond npix), 256 threads
__device__ __forceinline__ void stage_bwd_tile(float *tile, const float *base, const int64_t *st, int C, int W, int p0, int npix) {
    const int64_t sc = st[1], sh = st[2], sw = st[3];
    if (sc != 1) {
        for (int idx = threadIdx.x; idx < C * bwd::TILE_PIX; idx += blockDim.x) {
            const int pp = idx & 31, c = idx >> 5, p = p0 + pp;
            tile[c * 33 + pp] = pp < npix ? __ldg(base + c * sc + (p / W) * sh + (p % W) * sw) : 0.f;
        }
    } else {
        for (int idx = threadIdx.x; idx < C * bwd::TILE_PIX; idx += blockDim.x) {
            const int c = idx % C, pp = idx / C, p = p0 + pp;
            tile[c * 33 + pp] = pp < npix ? __ldg(base + c + (p / W) * sh + (p % W) * sw) : 0.f;
        }
    }
}

// DET = false: the default kernel, which scatters dL/dfeat_src with float atomics.  DET = true: the coefficient pass of the
// deterministic backward, the same operations up to the scatter, which it replaces by storing each sample's coefficients and
// folding the pixel's bound on its contributions into the pair's bound word.  (The switch is a parameter of the kernel itself:
// an inlined body function would allocate the default kernel's registers differently.)  vw: the views form, else empty.
template <int VEC, int NV, bool DET, typename... Views>
__global__ void __launch_bounds__(bwd::WARPS * 32) epi_fusion_bwd_kernel(const BwdArgs a, const Views... vw) {
    using namespace bwd;
    extern __shared__ float smem[];
    const int C = a.C, K = a.geom.K, H = a.geom.H, W = a.geom.W, HW = H * W;
    const int tiles_per_item = (HW + TILE_PIX - 1) / TILE_PIX;
    const int n = blockIdx.x / tiles_per_item;               // pair
    const PairItems it = bwd_items(n, vw...);                // its query and source items
    const int p0 = (blockIdx.x % tiles_per_item) * TILE_PIX;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int npix = min(TILE_PIX, HW - p0);
    float *q_tile = smem;                                    // [C][33]  query in, dL/dq out
    float *g_tile = smem + (size_t)C * 33;                   // [C][33]  dL/dout
    __shared__ PairGeom s_geom;
    if (tid == 0 && a.locs_in == nullptr) pair_geom_from_krt(a.P_ref + 12 * it.q, a.P_src + 12 * it.s, s_geom);

    auto stage_tile = [&](float *tile, const float *base, const int64_t *st) {
        const int64_t sc = st[1], sh = st[2], sw = st[3];
        if (sc != 1) {
            for (int idx = tid; idx < C * TILE_PIX; idx += blockDim.x) {
                const int pp = idx & 31, c = idx >> 5, p = p0 + pp;
                tile[c * 33 + pp] = pp < npix ? __ldg(base + c * sc + (p / W) * sh + (p % W) * sw) : 0.f;
            }
        } else {
            for (int idx = tid; idx < C * TILE_PIX; idx += blockDim.x) {
                const int c = idx % C, pp = idx / C, p = p0 + pp;
                tile[c * 33 + pp] = pp < npix ? __ldg(base + c + (p / W) * sh + (p % W) * sw) : 0.f;
            }
        }
    };
    stage_tile(q_tile, a.feat_ref + (int64_t)it.q * a.ref_stride[0], a.ref_stride);
    stage_tile(g_tile, a.grad_out + (int64_t)n * a.gout_stride[0], a.gout_stride);
    __syncthreads();

    const PairGeom g = s_geom;
    const GeomCfg gc = a.geom;
    const float *src = a.src_nhwc + (size_t)it.s * HW * C;
    float *dsrc = a.dsrc_nhwc ? a.dsrc_nhwc + (size_t)it.s * HW * C : nullptr;

    unsigned warp_bound = 0u;                        // DET: bits of the largest M_i of the warp's pixels
    for (int pi = 0; pi < TILE_PIX / WARPS; pi++) {
        const int pp = warp * (TILE_PIX / WARPS) + pi;
        if (pp >= npix) break;                       // warp-uniform
        const int p = p0 + pp, py_i = p / W, px_i = p % W;
        float q[NV * VEC], go[NV * VEC], dq[NV * VEC];
#pragma unroll
        for (int j = 0; j < NV; j++)
#pragma unroll
            for (int v = 0; v < VEC; v++) {
                const int c = (j * 32 + lane) * VEC + v;
                q[j * VEC + v] = c < C ? q_tile[c * 33 + pp] : 0.f;
                go[j * VEC + v] = c < C ? g_tile[c * 33 + pp] : 0.f;
                dq[j * VEC + v] = 0.f;
            }
        float sx = 0.f, sy = 0.f, ex = 0.f, ey = 0.f;
        if (a.locs_in == nullptr)
            line_endpoints(g, gc, pix2coord(px_i, gc.ds, gc.r), pix2coord(py_i, gc.ds, gc.r), sx, sy, ex, ey);

        float my_gx[MAXKCH], my_gy[MAXKCH], my_a[MAXKCH], my_da[MAXKCH], my_ds[MAXKCH];   // lane holds sample k = j*32+lane
        bool my_masked[MAXKCH];
#pragma unroll
        for (int j = 0; j < MAXKCH; j++) { my_gx[j] = my_gy[j] = my_a[j] = my_da[j] = my_ds[j] = 0.f; my_masked[j] = true; }

        auto gather = [&](const Taps &t, float *s) {              // s = Σ_t w_t F[p_t]  (lane's channels)
#pragma unroll
            for (int i = 0; i < NV * VEC; i++) s[i] = 0.f;
            if (!t.any) return;
#pragma unroll
            for (int tap = 0; tap < 4; tap++) {
                const float w = t.w[tap];
                if (w != 0.f) {                                     // warp-uniform
                    const float *row = src + ((size_t)(t.y0 + (tap >> 1)) * W + t.x0 + (tap & 1)) * C;
#pragma unroll
                    for (int jj = 0; jj < NV; jj++) {
                        const int c0 = (jj * 32 + lane) * VEC;
                        if (c0 < C) {
#pragma unroll
                            for (int v = 0; v < VEC; v++) s[jj * VEC + v] = fmaf(w, __ldg(row + c0 + v), s[jj * VEC + v]);
                        }
                    }
                }
            }
        };

        // ---- pass 1: sim_k (mask), dL/da_k = g·s_k ----
#pragma unroll
        for (int j = 0; j < MAXKCH; j++) {
            if (j * 32 >= K) break;
            {
                const int k = j * 32 + lane;
                float gx = 0.f, gy = 0.f;
                if (k < K) {
                    if (a.locs_in) {
                        const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + p);
                        gx = l.x; gy = l.y;
                    } else {
                        const float t = (float)k / (float)(K - 1);
                        gx = img2grid_x(lerp_exact(sx, ex, t), gc);
                        gy = img2grid_y(lerp_exact(sy, ey, t), gc);
                    }
                    my_a[j] = __ldg(a.attn + ((size_t)n * K + k) * HW + p);
                    if (a.grad_attn) my_da[j] = __ldg(a.grad_attn + ((size_t)n * K + k) * HW + p);
                }
                my_gx[j] = gx; my_gy[j] = gy;
            }
            const int kend = min(32, K - j * 32);
            for (int kk = 0; kk < kend; kk++) {
                const Taps t = make_taps(__shfl_sync(0xffffffffu, my_gx[j], kk), __shfl_sync(0xffffffffu, my_gy[j], kk), H, W, gc.align);
                float s[NV * VEC];
                gather(t, s);
                float sim = 0.f, da = 0.f;
#pragma unroll
                for (int i = 0; i < NV * VEC; i++) { sim = fmaf(s[i], q[i], sim); da = fmaf(s[i], go[i], da); }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) { sim += __shfl_xor_sync(0xffffffffu, sim, o); da += __shfl_xor_sync(0xffffffffu, da, o); }
                if (lane == kk) { my_masked[j] = (sim == 0.f); my_da[j] += da; }
            }
        }
        // ---- softmax backward ----
        float dot = 0.f;
#pragma unroll
        for (int j = 0; j < MAXKCH; j++) if (j * 32 < K) dot = fmaf(my_a[j], my_da[j], dot);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
#pragma unroll
        for (int j = 0; j < MAXKCH; j++)
            if (j * 32 < K) my_ds[j] = (my_masked[j] || j * 32 + lane >= K) ? 0.f : a.softmax_scale * my_a[j] * (my_da[j] - dot);
        if constexpr (DET) {
            // cv_k / ck_k as the scatter would use them, and M_i = Σ over the samples it would scatter of |cv_k|·‖g‖∞ + |ck_k|·‖q‖∞.
            // The norms are maxima of |x|'s bits, under which a NaN ranks above +inf, so a non-finite map or gradient value
            // makes M_i non-finite.
            unsigned gb = 0u, qb = 0u;
#pragma unroll
            for (int i = 0; i < NV * VEC; i++) { gb = max(gb, __float_as_uint(fabsf(go[i]))); qb = max(qb, __float_as_uint(fabsf(q[i]))); }
            const float gmax = __uint_as_float(__reduce_max_sync(0xffffffffu, gb)), qmax = __uint_as_float(__reduce_max_sync(0xffffffffu, qb));
            float bound = 0.f;
#pragma unroll
            for (int j = 0; j < MAXKCH; j++) {
                const int k = j * 32 + lane;
                if (j * 32 >= K || k >= K) continue;
                const float cv = a.grad_vals ? my_a[j] : 0.f, ck = a.grad_keys ? my_ds[j] : 0.f;
                a.coef[((size_t)n * K + k) * HW + p] = make_float2(cv, ck);
                if ((cv != 0.f || ck != 0.f) && make_taps(my_gx[j], my_gy[j], H, W, gc.align).any) bound += fabsf(cv) * gmax + fabsf(ck) * qmax;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) bound += __shfl_xor_sync(0xffffffffu, bound, o);
            warp_bound = max(warp_bound, __float_as_uint(fabsf(bound)));
        }

        // ---- pass 2: dL/dq and the scatter into dL/dF ----
#pragma unroll
        for (int j = 0; j < MAXKCH; j++) {
            if (j * 32 >= K) break;
            const int kend = min(32, K - j * 32);
            for (int kk = 0; kk < kend; kk++) {
                const float ak = __shfl_sync(0xffffffffu, my_a[j], kk), ds = __shfl_sync(0xffffffffu, my_ds[j], kk);
                const Taps t = make_taps(__shfl_sync(0xffffffffu, my_gx[j], kk), __shfl_sync(0xffffffffu, my_gy[j], kk), H, W, gc.align);
                if (!t.any) continue;
                const float cv = a.grad_vals ? ak : 0.f, ck = a.grad_keys ? ds : 0.f;
                if (ds != 0.f) {
                    float s[NV * VEC];
                    gather(t, s);
#pragma unroll
                    for (int i = 0; i < NV * VEC; i++) dq[i] = fmaf(ds, s[i], dq[i]);
                }
                if (!DET && dsrc && (cv != 0.f || ck != 0.f)) {
#pragma unroll
                    for (int tap = 0; tap < 4; tap++) {
                        const float w = t.w[tap];
                        if (w != 0.f) {
                            float *row = dsrc + ((size_t)(t.y0 + (tap >> 1)) * W + t.x0 + (tap & 1)) * C;
#pragma unroll
                            for (int jj = 0; jj < NV; jj++) {
                                const int c0 = (jj * 32 + lane) * VEC;
                                if (c0 < C) {
                                    float v[VEC];
#pragma unroll
                                    for (int e = 0; e < VEC; e++) v[e] = w * fmaf(cv, go[jj * VEC + e], ck * q[jj * VEC + e]);
                                    if (VEC == 4) atomicAdd(reinterpret_cast<float4 *>(row + c0), make_float4(v[0], v[1], v[2], v[3]));
                                    else
#pragma unroll
                                        for (int e = 0; e < VEC; e++) atomicAdd(row + c0 + e, v[e]);
                                }
                            }
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < NV; j++)
#pragma unroll
            for (int v = 0; v < VEC; v++) {
                const int c = (j * 32 + lane) * VEC + v;
                if (c < C) q_tile[c * 33 + pp] = dq[j * VEC + v];
            }
    }
    if (DET && lane == 0 && warp_bound != 0u) atomicMax(a.pair_max + it.s, warp_bound);   // max of non-negative floats: their bits' max
    __syncthreads();
    if (a.grad_ref) {
        float *obase = a.grad_ref + (int64_t)n * a.gref_stride[0];
        const int64_t sc = a.gref_stride[1], sh = a.gref_stride[2], sw = a.gref_stride[3];
        if (sc != 1) {
            for (int idx = tid; idx < C * TILE_PIX; idx += blockDim.x) {
                const int pp = idx & 31, c = idx >> 5, p = p0 + pp;
                if (pp < npix) obase[c * sc + (p / W) * sh + (p % W) * sw] = q_tile[c * 33 + pp];
            }
        } else {
            for (int idx = tid; idx < C * TILE_PIX; idx += blockDim.x) {
                const int c = idx % C, pp = idx / C, p = p0 + pp;
                if (pp < npix) obase[c + (p / W) * sh + (p % W) * sw] = q_tile[c * 33 + pp];
            }
        }
    }
}

// Fixed-point scatter of the deterministic backward: one warp per reference pixel, tiled like the coefficient pass.  It re-derives
// each sample's taps as pass 1 does (from locs_in or the cameras, with the same functions), forms every contribution in fp32 as the
// default scatter does, and adds round(v·2^s) to the int64 accumulator.  Integer addition is associative, so the sums do not
// depend on the order the warps' atomics land in.  A pair with a zero or non-finite bound adds nothing.
template <int VEC, int NV, typename... Views>
__global__ void __launch_bounds__(bwd::WARPS * 32) epi_fusion_bwd_scatter_kernel(const BwdArgs a, const Views... vw) {
    using namespace bwd;
    extern __shared__ float smem[];
    const int C = a.C, K = a.geom.K, H = a.geom.H, W = a.geom.W, HW = H * W;
    const int tiles_per_item = (HW + TILE_PIX - 1) / TILE_PIX;
    const int n = blockIdx.x / tiles_per_item;                       // pair
    const PairItems it = bwd_items(n, vw...);                        // its query and source items
    const int p0 = (blockIdx.x % tiles_per_item) * TILE_PIX;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int npix = min(TILE_PIX, HW - p0);
    int s;
    if (!bwd_scale(__ldg(a.pair_max + it.s), HW, it.s, s, vw...)) return;    // block-uniform
    const double scale = ldexp(1.0, s);                              // exact in fp64 for every s a float bound can give
    float *q_tile = smem;                                            // [C][33]  query
    float *g_tile = smem + (size_t)C * 33;                           // [C][33]  dL/dout
    __shared__ PairGeom s_geom;
    if (tid == 0 && a.locs_in == nullptr) pair_geom_from_krt(a.P_ref + 12 * it.q, a.P_src + 12 * it.s, s_geom);
    stage_bwd_tile(q_tile, a.feat_ref + (int64_t)it.q * a.ref_stride[0], a.ref_stride, C, W, p0, npix);
    stage_bwd_tile(g_tile, a.grad_out + (int64_t)n * a.gout_stride[0], a.gout_stride, C, W, p0, npix);
    __syncthreads();

    const PairGeom g = s_geom;
    const GeomCfg gc = a.geom;
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(a.acc) + (size_t)it.s * HW * C;   // two's complement sums
    for (int pi = 0; pi < TILE_PIX / WARPS; pi++) {
        const int pp = warp * (TILE_PIX / WARPS) + pi;
        if (pp >= npix) break;                       // warp-uniform
        const int p = p0 + pp, py_i = p / W, px_i = p % W;
        float q[NV * VEC], go[NV * VEC];
#pragma unroll
        for (int j = 0; j < NV; j++)
#pragma unroll
            for (int v = 0; v < VEC; v++) {
                const int c = (j * 32 + lane) * VEC + v;
                q[j * VEC + v] = c < C ? q_tile[c * 33 + pp] : 0.f;
                go[j * VEC + v] = c < C ? g_tile[c * 33 + pp] : 0.f;
            }
        float sx = 0.f, sy = 0.f, ex = 0.f, ey = 0.f;
        if (a.locs_in == nullptr)
            line_endpoints(g, gc, pix2coord(px_i, gc.ds, gc.r), pix2coord(py_i, gc.ds, gc.r), sx, sy, ex, ey);
        for (int j = 0; j < MAXKCH; j++) {
            if (j * 32 >= K) break;
            const int k = j * 32 + lane;
            float gx = 0.f, gy = 0.f;
            float2 cf = make_float2(0.f, 0.f);
            if (k < K) {
                if (a.locs_in) {
                    const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + p);
                    gx = l.x; gy = l.y;
                } else {
                    const float t = (float)k / (float)(K - 1);
                    gx = img2grid_x(lerp_exact(sx, ex, t), gc);
                    gy = img2grid_y(lerp_exact(sy, ey, t), gc);
                }
                cf = __ldg(a.coef + ((size_t)n * K + k) * HW + p);
            }
            const int kend = min(32, K - j * 32);
            for (int kk = 0; kk < kend; kk++) {
                const float cv = __shfl_sync(0xffffffffu, cf.x, kk), ck = __shfl_sync(0xffffffffu, cf.y, kk);
                const Taps t = make_taps(__shfl_sync(0xffffffffu, gx, kk), __shfl_sync(0xffffffffu, gy, kk), H, W, gc.align);
                if (!t.any || (cv == 0.f && ck == 0.f)) continue;
#pragma unroll
                for (int tap = 0; tap < 4; tap++) {
                    const float w = t.w[tap];
                    if (w != 0.f) {
                        unsigned long long *row = acc + ((size_t)(t.y0 + (tap >> 1)) * W + t.x0 + (tap & 1)) * C;
#pragma unroll
                        for (int jj = 0; jj < NV; jj++) {
                            const int c0 = (jj * 32 + lane) * VEC;
                            if (c0 < C) {
#pragma unroll
                                for (int e = 0; e < VEC; e++) {
                                    const float v = w * fmaf(cv, go[jj * VEC + e], ck * q[jj * VEC + e]);
                                    atomicAdd(row + c0 + e, (unsigned long long)__double2ll_rn((double)v * scale));
                                }
                            }
                        }
                    }
                }
            }
        }
    }
}

template <int VEC, int NV, typename... Views>
static cudaError_t launch_bwd_t(const BwdArgs &a, cudaStream_t st, bool det, const Views &...vw) {
    const int HW = a.geom.H * a.geom.W;
    const int tiles = (HW + bwd::TILE_PIX - 1) / bwd::TILE_PIX;
    const size_t smem = (size_t)a.C * 33 * 2 * sizeof(float);
    // (each entry a conditional: a kernel template with a trailing parameter pack converts to a pointer only once it is resolved)
    void (*const kernels[2])(const BwdArgs, const Views...) = {det ? epi_fusion_bwd_kernel<VEC, NV, true, Views...> : epi_fusion_bwd_kernel<VEC, NV, false, Views...>,
                                                               det ? epi_fusion_bwd_scatter_kernel<VEC, NV, Views...> : nullptr};
    for (int i = 0; i < (det ? 2 : 1); i++) {
        cudaError_t e = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kernels[i]<<<a.N * tiles, bwd::WARPS * 32, smem, st>>>(a, vw...);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <typename... Views>
static cudaError_t launch_bwd(const BwdArgs &a, cudaStream_t st, bool det, const Views &...vw) {
    const int C = a.C;
    if (C % 4 == 0 && C <= 128) return launch_bwd_t<4, 1>(a, st, det, vw...);
    if (C % 4 == 0 && C <= 256) return launch_bwd_t<4, 2>(a, st, det, vw...);
    if (C % 4 == 0 && C <= 512) return launch_bwd_t<4, 4>(a, st, det, vw...);
    if (C <= 32) return launch_bwd_t<1, 1>(a, st, det, vw...);
    if (C <= 128) return launch_bwd_t<1, 4>(a, st, det, vw...);
    return cudaErrorInvalidValue;
}

cudaError_t launch_fusion_bwd(const BwdArgs &a, cudaStream_t st) { return launch_bwd(a, st, false); }

cudaError_t launch_fusion_bwd_det(const BwdArgs &a, cudaStream_t st, int &launched) {
    const cudaError_t e = launch_bwd(a, st, true);
    launched = e == cudaSuccess ? 2 : 0;
    return e;
}

cudaError_t launch_fusion_bwd_views(const BwdArgs &a, const BwdViews &vw, cudaStream_t st, bool det, int &launched) {
    const cudaError_t e = launch_bwd(a, st, det, vw);
    launched = e == cudaSuccess ? (det ? 2 : 1) : 0;
    return e;
}

}  // namespace epi
