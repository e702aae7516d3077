// epi_stage.cu — the ONE operand-staging launch in front of the fused attention kernel (epi_fusion_pipe.cu):
//
//   blocks [0, N)      per (ref, src) pair (pair n: items pair_items(n, n_ref, n_views, vs), epi_common.cuh): fp64 pair constants (camera centre, epipole, infinite homography;
//                      /root/reference/vision/multiview.py:16-21, modeling/layers/epipolar.py:336-348) and the list of
//                      reference pixels sorted by epipolar angle (counting sort on a 12-bit angle key, ties by pixel index
//                      => deterministic).  Pixels on one epipolar line of the reference view share one epipolar line in
//                      the source view, so 32 consecutive list entries have nearly identical sets of bilinear taps.
//   remaining blocks   [N,C,H,W] (any strides; fp32, bf16 or fp16 elements) -> pixel-major bf16 (hi, lo) planes [N,H*W,C] with
//                      x ≈ hi + lo, for BOTH feature maps (reference -> planes 0,1; source -> planes 2,3 of one buffer), 64 x 64
//                      tiles through shared memory: coalesced 4-pixel vector reads along pixels, 16-byte writes along channels.
//                      The reference map has n_ref items and the source map N (several source views per reference item:
//                      N = S·n_ref), so a reference tile is staged once however many sources it is fused with.  In the views
//                      form (n_views = V) the reference map holds the V·n_ref view items and is the only map: each view is
//                      staged once and serves as the query of its S pairs (S = V−1, or the source table's width) and the
//                      source of whichever pairs name it.
//                      fp16 values are split exactly like fp32 ones (hi + lo holds them exactly); a bf16 value is its own hi
//                      part, so bf16 maps write hi planes only (reference -> plane 0, source -> plane 1).
// Also zeroes the fused kernel's tile counter and error word.
#include <cuda_bf16.h>

#include <type_traits>

#include "epi_kernels.cuh"

namespace epi {

namespace stg {
constexpr int NT = 256;
constexpr int NBIN = 4096;
constexpr int SMALL = 32;
constexpr int TC = 64, TPX = 64, TPITCH = 65;       // layout-staging tile: 64 channels x 64 pixels (stage_planes_tile's)

// Monotone pseudo-angle of (u, v) in [-2, 2] (diamond angle): same ordering as atan2(v, u) at the price of one division.
__device__ __forceinline__ float pseudo_angle(float u, float v) {
    const float p = __fdividef(v, fabsf(u) + fabsf(v) + 1e-30f);
    return u >= 0.f ? p : (v >= 0.f ? 2.f - p : -2.f - p);
}
// key in [0,1): position of the pixel centre (px, py) inside the image's span [lo, lo + 1/inv_span] of the pseudo-angle
// around the epipole, measured from the direction (cdx, cdy) epipole -> image centre (so the cut lies behind the epipole);
// for an epipole at infinity: the offset across the parallel epipolar lines of direction (cdx, cdy)
__device__ __forceinline__ float angle_key(float px, float py, float ex, float ey, float cdx, float cdy, bool parallel, float lo, float inv_span) {
    float u;
    if (parallel) u = (px * (-cdy) + py * cdx - lo) * inv_span;
    else {
        const float dx = px - ex, dy = py - ey;
        u = (pseudo_angle(dx * cdx + dy * cdy, dy * cdx - dx * cdy) - lo) * inv_span;
    }
    u = fminf(fmaxf(u, 0.f), 0.99999f);
    if (!(u == u)) u = 0.f;
    return u;
}
}  // namespace stg

#ifdef EPI_PIPE_TIMERS
__device__ unsigned long long g_stage_timers[16];
#define ST(slot) do { __syncthreads(); if (t == 0 && blockIdx.x == 0) { const long long t_ = clock64(); g_stage_timers[slot] = (unsigned long long)(t_ - st_prev); st_prev = t_; } } while (0)
extern "C" void epi_stage_timers_read(unsigned long long *out16) { cudaMemcpyFromSymbol(out16, g_stage_timers, sizeof(unsigned long long) * 16); }
#else
#define ST(slot) do { } while (0)
#endif

template <typename T>
struct StageArgs {
    const T *ref, *src;
    int64_t ref_stride[4], src_stride[4];
    __nv_bfloat16 *planes;            // ref_hi, ref_lo [n_ref*HW][C], src_hi, src_lo [N*HW][C]  (bf16 maps: ref_hi, src_hi)
    const float *P_ref, *P_src;       // may be null (injected locations): no order, no pair constants
    PairGeom *pair_geom;              // [N]
    uint16_t *order;                  // [N][HW]
    int *zero_words;                  // tile counter, error word
    float *order_key;                 // optional [N][32]: key of the cached (order, pair constants); null = rebuild every call
    const float *Wf;                  // optional [C][C] folded z weight -> bf16 (hi, lo) planes w_planes [2][C][C]
    int w_add_identity;               // ZRESIDUAL folded into the weight: planes hold Wf + I
    __nv_bfloat16 *w_planes;
    int N, C, H, W;
    int n_ref, n_views;               // pair n reads items pair_items(n, n_ref, n_views[, vs])
    int ref_tiles;                    // layout tiles of the reference map (n_ref items, or n_views·n_ref); the source map has N items
    size_t ref_elems;                 // elements of one reference plane
    size_t src_plane0;                // offset of the source hi plane in `planes`
    int do_ref, do_src, do_order;
    int persist;                      // > 0: whole vectorisable tiles only -> `persist` streaming blocks loop over the tiles
    GeomCfg gc;
};

// (min 5 blocks per SM: the layout-staging blocks need few registers; the rare order blocks may spill a little)
// MULTI: several source views per reference item (n_ref < N), or the views form.  The one-source instantiation keeps the single-map-size indexing,
// so its code (and its register allocation, tight at 48 registers) does not pay for the general mapping.
// vs: the source table of a table call, else empty (pair_items)
template <typename T, bool MULTI, typename... Tab>
__global__ void __launch_bounds__(stg::NT, 5) epi_stage_kernel(const StageArgs<T> s, const Tab... vs) {
    using namespace stg;
    constexpr bool LO = !std::is_same<T, __nv_bfloat16>::value;   // a bf16 value's lo part is zero: no lo planes
    constexpr int NPL = LO ? 2 : 1;                               // planes per map
    extern __shared__ __align__(16) uint8_t dyn[];        // transposition tile [64 ch][65] fp32 | order blocks: histogram + pixel list
    float (*tile)[TPITCH] = reinterpret_cast<float (*)[TPITCH]>(dyn);
    const int t = threadIdx.x;
    const int H = s.H, W = s.W, HW = H * W, C = s.C;
    const int nord = s.do_order ? s.N : 0;
    pdl_launch_dependents();                               // the fused kernel's CTAs may start their prologue as SMs drain
    pdl_wait();                                            // previous forward's kernels (they read what this launch rewrites)
    if (blockIdx.x == 0 && t == 0 && s.zero_words) { s.zero_words[0] = 0; s.zero_words[1] = 0; }

    if ((int)blockIdx.x < nord) {
        // ------------------------------------------------------------------------------------------------
        // pair constants + epipolar-angle order of the pair's reference pixels
        // ------------------------------------------------------------------------------------------------
        int *hist = reinterpret_cast<int *>(dyn);                      // NBIN counts -> offsets
        uint16_t *lst = reinterpret_cast<uint16_t *>(dyn + NBIN * 4);  // [HW] pixels grouped by bin (then sorted inside each bin)
        __shared__ float s_e[8];                                  // [7]: cache hit
        __shared__ int s_warp[NT / 32];
        __shared__ int s_big[64], s_nbig;
#ifdef EPI_PIPE_TIMERS
        long long st_prev = clock64();
#endif
        const int n = blockIdx.x;                                        // pair
        const PairItems pi = MULTI ? pair_items(n, s.n_ref, s.n_views, vs...) : PairItems{n, n};
        // cached order: the key is (P_ref, P_src, geometry configuration); an unchanged camera pair costs 32 compares
        float my_key = 0.f;
        if (t < 32) {
            if (t < 12) my_key = s.P_ref[12 * pi.q + t];
            else if (t < 24) my_key = s.P_src[12 * pi.s + t - 12];
            else if (t == 24) my_key = (float)H;
            else if (t == 25) my_key = (float)W;
            else if (t == 26) my_key = s.gc.ds;
            else if (t == 27) my_key = s.gc.r;
            else if (t == 28) my_key = 1.f;                      // valid marker (a zero-initialised cache never matches)
            else if (t == 29) my_key = (float)(s.gc.K + 1024 * s.gc.correct + 2048 * s.gc.align);
            else if (t == 30) my_key = s.gc.eps;
            // slot 31 = epoch of this pair's cached plan (bumped on every miss; read by the fused kernel), not part of the comparison
            if (s.order_key) {
                const bool same = t == 31 || __float_as_uint(s.order_key[32 * n + t]) == __float_as_uint(my_key);
                if (__all_sync(0xffffffffu, same)) s_e[7] = 1.f; else s_e[7] = 0.f;
            } else s_e[7] = 0.f;
        }
        __syncthreads();
        if (s_e[7] != 0.f) return;                               // hit: order and pair constants are already in place
        if (t == 0) {
            const float *P1 = s.P_ref + 12 * pi.q, *P2 = s.P_src + 12 * pi.s;
            PairGeom g;
            pair_geom_from_krt(P1, P2, g);
            s.pair_geom[n] = g;
            // epipole of the SOURCE camera in the reference view: e1 = P_ref·[C_src; 1]
            double a[9], t1[3], b[9], t2[3], bi[9], cs[3], e[3];
            cam_load(P2, b, t2);
            cam_inverse(b, bi);
            cam_centre(bi, t2, cs);
            cam_load(P1, a, t1);
            for (int r = 0; r < 3; r++) e[r] = cam_project(a, t1, cs, r);
            const double cx = 0.5 * ((double)s.gc.xmin + s.gc.xmax), cy = 0.5 * ((double)s.gc.ymin + s.gc.ymax);
            const double nrm = fabs(e[0]) + fabs(e[1]) + 1e-300;
            // range of the key over the image: the four corners bound it unless the epipole lies inside the image
            const float cxs[4] = {s.gc.xmin, s.gc.xmax, s.gc.xmin, s.gc.xmax}, cys[4] = {s.gc.ymin, s.gc.ymin, s.gc.ymax, s.gc.ymax};
            float lo = 1e30f, hi = -1e30f, exf = 0.f, eyf = 0.f, cdx, cdy, par;
            if (!(fabs(e[2]) > 1e-9 * nrm)) {        // epipole at infinity (or NaN): parallel lines, sort by the offset across them
                cdx = (float)(e[0] / nrm); cdy = (float)(e[1] / nrm); par = 1.f;
                for (int q = 0; q < 4; q++) { const float v = cxs[q] * (-cdy) + cys[q] * cdx; lo = fminf(lo, v); hi = fmaxf(hi, v); }
            } else {
                const double ex = e[0] / e[2], ey = e[1] / e[2];
                const double dn = sqrt((cx - ex) * (cx - ex) + (cy - ey) * (cy - ey)) + 1e-300;
                exf = (float)ex; eyf = (float)ey; cdx = (float)((cx - ex) / dn); cdy = (float)((cy - ey) / dn); par = 0.f;
                const bool inside = ex >= s.gc.xmin && ex <= s.gc.xmax && ey >= s.gc.ymin && ey <= s.gc.ymax;
                if (inside) { lo = -2.f; hi = 2.f; }
                else
                    for (int q = 0; q < 4; q++) {
                        const float dx = cxs[q] - exf, dy = cys[q] - eyf;
                        const float v = pseudo_angle(dx * cdx + dy * cdy, dy * cdx - dx * cdy);
                        lo = fminf(lo, v); hi = fmaxf(hi, v);
                    }
            }
            if (!(hi > lo)) { lo = 0.f; hi = 1.f; }
            s_e[0] = exf; s_e[1] = eyf; s_e[2] = cdx; s_e[3] = cdy; s_e[4] = par; s_e[5] = lo; s_e[6] = 1.f / ((hi - lo) * 1.0001f + 1e-20f);
            s_nbig = 0;
        }
        for (int b = t; b < NBIN; b += NT) hist[b] = 0;
        __syncthreads();
        ST(0);
        const float ex = s_e[0], ey = s_e[1], cdx = s_e[2], cdy = s_e[3], klo = s_e[5], kinv = s_e[6];
        const bool parallel = s_e[4] != 0.f;
        // bins of this thread's pixels (i = t + 256 m), kept in registers between the two passes (maps up to 16384 pixels; larger
        // maps recompute the key in the placement pass — the order is cached per camera pair, so this runs once per rig)
        constexpr int MAXPT = 64;
        const int npt = (HW - t + NT - 1) / NT;
        const bool keep = npt <= MAXPT;
        uint16_t bins[MAXPT];
        auto bin_of = [&](int x, int y) -> int {
            return (int)(angle_key(pix2coord(x, s.gc.ds, s.gc.r), pix2coord(y, s.gc.ds, s.gc.r), ex, ey, cdx, cdy, parallel, klo, kinv) * (float)NBIN);
        };
        const int sx = NT % W, sy = NT / W;
        if (keep) {
            int x = t % W, y = t / W;
#pragma unroll 4
            for (int m = 0; m < MAXPT; m++) {
                if (m < npt) {
                    const int b = bin_of(x, y);
                    bins[m] = (uint16_t)b;
                    atomicAdd(&hist[b], 1);
                    x += sx; y += sy;
                    if (x >= W) { x -= W; y++; }
                }
            }
        } else {
            int x = t % W, y = t / W;
            for (int m = 0; m < npt; m++) {
                atomicAdd(&hist[bin_of(x, y)], 1);
                x += sx; y += sy;
                if (x >= W) { x -= W; y++; }
            }
        }
        __syncthreads();
        ST(1);
        // exclusive scan over the bins: 16 consecutive bins per thread, then a block scan of the partial sums
        constexpr int PER = NBIN / NT;
        int loc[PER], sum = 0;
#pragma unroll
        for (int q = 0; q < PER; q++) { loc[q] = hist[t * PER + q]; sum += loc[q]; }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if ((t & 31) >= o) incl += v; }
        if ((t & 31) == 31) s_warp[t >> 5] = incl;
        __syncthreads();
        int base = incl - sum;
        for (int w = 0; w < (t >> 5); w++) base += s_warp[w];
        const int start0 = base;
        __syncthreads();
#pragma unroll
        for (int q = 0; q < PER; q++) { hist[t * PER + q] = base; base += loc[q]; }
        __syncthreads();
        ST(2);
        // placement (arbitrary order inside a bin) into the shared list
        if (keep) {
#pragma unroll 4
            for (int m = 0; m < MAXPT; m++)
                if (m < npt) lst[atomicAdd(&hist[bins[m]], 1)] = (uint16_t)(t + NT * m);
        } else {
            int x = t % W, y = t / W;
            for (int m = 0; m < npt; m++) {
                lst[atomicAdd(&hist[bin_of(x, y)], 1)] = (uint16_t)(t + NT * m);
                x += sx; y += sy;
                if (x >= W) { x -= W; y++; }
            }
        }
        __syncthreads();
        ST(3);
        // inside every bin: ascending pixel index (in-place insertion sort; bins hold ~HW/4096 entries)
        uint16_t *ord = s.order + (size_t)n * HW;
        {
            int st0 = start0;
#pragma unroll
            for (int q = 0; q < PER; q++) {
                const int len = loc[q];
                bool coop = false;                          // long bins are ranked by the whole block below (64 of them at most)
                if (len > (keep ? SMALL : 4 * SMALL)) {
                    const int slot = atomicAdd(&s_nbig, 1);
                    if (slot < 64) { s_big[slot] = t * PER + q; coop = true; }
                }
                if (!coop) {
                    for (int e = 1; e < len; e++) {
                        const uint16_t xv = lst[st0 + e];
                        int p = e;
                        while (p > 0 && lst[st0 + p - 1] > xv) { lst[st0 + p] = lst[st0 + p - 1]; p--; }
                        lst[st0 + p] = xv;
                    }
                }
                st0 += len;
            }
        }
        __syncthreads();
        ST(4);
        const int nbig = s_nbig < 64 ? s_nbig : 64;
        for (int i = t; i < HW; i += NT) ord[i] = lst[i];
        // degenerate cameras only: big bins are ranked by counting (unique values), the whole block per bin, straight to global
        for (int bb = 0; bb < nbig; bb++) {
            const int b = s_big[bb];
            const int end = hist[b], beg = b == 0 ? 0 : hist[b - 1];     // after placement hist[b] = end of bin b
            __syncthreads();
            for (int e = beg + t; e < end; e += NT) {
                const uint16_t xv = lst[e];
                int r = 0;
                for (int f = beg; f < end; f++) r += lst[f] < xv;
                ord[beg + r] = xv;
            }
        }
        if (s.order_key) {                                       // publish the key last (same stream => ordered for the next call)
            __syncthreads();
            if (t < 31) s.order_key[32 * n + t] = my_key;
            else if (t == 31) reinterpret_cast<uint32_t *>(s.order_key)[32 * n + 31] += 1u;   // invalidates the pair's cached work items
        }
        return;
    }

    // ----------------------------------------------------------------------------------------------------
    // layout staging: 64 channels x 64 pixels per block
    // ----------------------------------------------------------------------------------------------------
    const int tiles_p = (HW + TPX - 1) / TPX, tiles_c = (C + TC - 1) / TC;
    const int src_tiles = MULTI && !s.do_src ? 0 : tiles_p * tiles_c * s.N, ref_tiles = MULTI ? s.ref_tiles : src_tiles;
    int lin = (int)blockIdx.x - nord;
    const int wblocks = (s.Wf && s.w_planes) ? (C * C / 8 + NT - 1) / NT : 0;
    // block roles after the order blocks: [tiles | weight blocks], or with streaming blocks [weight blocks | streaming blocks]
    const int wlin = s.persist ? lin : lin - (ref_tiles + src_tiles);
    if (wlin >= 0 && wlin < wblocks) {
        // folded z weight [C out][C in] fp32 -> bf16 (hi, lo) planes (B operand of the z GEMM), 8 elements per thread
        const size_t e0 = ((size_t)wlin * NT + t) * 8, tot = (size_t)C * C;
        if (e0 < tot) {
            const float4 a4 = __ldg(reinterpret_cast<const float4 *>(s.Wf + e0)), b4 = __ldg(reinterpret_cast<const float4 *>(s.Wf + e0 + 4));
            float f[8] = {a4.x, a4.y, a4.z, a4.w, b4.x, b4.y, b4.z, b4.w};
            if (s.w_add_identity) {                           // y = Wf·x + x  ==  (Wf + I)·x : the ZRESIDUAL costs nothing in the GEMM
                const int o = (int)(e0 / C), c_first = (int)(e0 % C);
                if (o >= c_first && o < c_first + 8) f[o - c_first] += 1.f;
            }
            uint4 h4, l4;
            split8(f, h4, l4);
            *reinterpret_cast<uint4 *>(s.w_planes + e0) = h4;
            *reinterpret_cast<uint4 *>(s.w_planes + tot + e0) = l4;
        }
        return;
    }
    constexpr int QW = TPX / 4, RPP = NT / QW, RPASS = TC / RPP;        // float4 per channel row, channel rows per pass, passes
    // ---- whole NCHW tiles ----
    // Fast path (whole NCHW tile): the (hi, lo) split happens BEFORE the transposition, on bf16x2 words of two adjacent channels,
    // so shared memory carries 2 x 8 KB of 32-bit words instead of 16 KB of fp32 scalars.  Half-warps load 256-byte rows of two
    // adjacent channels and swap halves (lanes < 16 keep pixels 4q, 4q+1; lanes >= 16 pixels 4q+2, 4q+3).  Word (px, cpair) lives at
    // row px, position ((g ^ a) << 2) | (k ^ b) with g = cpair / 4, k = cpair % 4, (a, b) = bits of px / 2: the 32 lanes of a
    // store (one channel pair, 32 pixels of one parity) hit 32 different banks, and the 16-byte reads of a pixel's 8 channel groups
    // cover its whole 128-byte row; the reader undoes the k ^ b order with four selects.
    uint32_t *whi = reinterpret_cast<uint32_t *>(dyn), *wlo = whi + TPX * 32;
    const int fq = t & 15, hsel = (t >> 4) & 1, fw = t >> 5;
    auto fast_load = [&](const T *spn, int64_t scn, int c0n, int p0n, float4 *v) {
#pragma unroll
        for (int i = 0; i < RPASS; i++) v[i] = ld4_cs(spn + (int64_t)(c0n + 2 * fw + hsel + i * RPP) * scn + p0n + fq * 4);   // read once: streaming, keeps L2 for the planes
    };
    auto fast_split = [&](const float4 *v) {            // registers -> (hi, lo) words in shared memory
#pragma unroll
        for (int i = 0; i < RPASS; i++) {
            const float sx = hsel ? v[i].x : v[i].z, sy = hsel ? v[i].y : v[i].w;          // what the partner lane needs
            const float rx = __shfl_xor_sync(0xffffffffu, sx, 16), ry = __shfl_xor_sync(0xffffffffu, sy, 16);
            // pixel pair of this lane: even channel first
            const float e0 = hsel ? rx : v[i].x, o0 = hsel ? v[i].z : rx;                   // pixel 4q + 2 hsel
            const float e1 = hsel ? ry : v[i].y, o1 = hsel ? v[i].w : ry;                   // pixel 4q + 2 hsel + 1
            const int cpair = fw + 8 * i, g = cpair >> 2, k = cpair & 3;
#pragma unroll
            for (int u = 0; u < 2; u++) {
                uint32_t hw, lw;
                split_bf16x2(u ? e1 : e0, u ? o1 : o0, hw, lw);
                const int px = 4 * fq + 2 * hsel + u, sw5 = (px >> 1) & 31;
                const int pos = px * 32 + (((g ^ (sw5 >> 2)) << 2) | (k ^ (sw5 & 3)));
                whi[pos] = hw;
                if (LO) wlo[pos] = lw;
            }
        }
    };
    auto fast_store = [&](__nv_bfloat16 *hin, __nv_bfloat16 *lon, int nn, int c0n, int p0n) {     // shared memory -> pixel-major planes
        const int g = t & 7, pl = t >> 3;
#pragma unroll
        for (int i = 0; i < TPX / (NT / 8); i++) {
            const int px = pl + i * (NT / 8), sw5 = (px >> 1) & 31;
            const int pos = px * 32 + ((g ^ (sw5 >> 2)) << 2);
            uint4 h4 = *reinterpret_cast<const uint4 *>(whi + pos), l4 = *reinterpret_cast<const uint4 *>(wlo + pos);
            if (sw5 & 1) { uint32_t x_; x_ = h4.x; h4.x = h4.y; h4.y = x_; x_ = h4.z; h4.z = h4.w; h4.w = x_; x_ = l4.x; l4.x = l4.y; l4.y = x_; x_ = l4.z; l4.z = l4.w; l4.w = x_; }
            if (sw5 & 2) { uint32_t x_; x_ = h4.x; h4.x = h4.z; h4.z = x_; x_ = h4.y; h4.y = h4.w; h4.w = x_; x_ = l4.x; l4.x = l4.z; l4.z = x_; x_ = l4.y; l4.y = l4.w; l4.w = x_; }
            const size_t o = ((size_t)nn * HW + p0n + px) * C + c0n + g * 8;
            *reinterpret_cast<uint4 *>(hin + o) = h4;
            if (LO) *reinterpret_cast<uint4 *>(lon + o) = l4;
        }
    };
    // reference and source tiles alternate while both remain (see below); the source tiles of the further sources follow
    // (tile index l -> map, tile of that map)
    auto split_tile = [&](int &l) -> int {
        if (MULTI && !s.do_src) return 0;                               // the views form: one map
        if (!MULTI || l < 2 * ref_tiles) { const int mp = l & 1; l >>= 1; return mp; }
        l -= ref_tiles;
        return 1;
    };
    const size_t plane_elems_all = (size_t)s.N * HW * C;                 // one source plane (= one reference plane unless MULTI)
    auto plane_hi = [&](int mp) { return MULTI ? s.planes + (mp ? s.src_plane0 : (size_t)0) : s.planes + (size_t)(NPL * mp) * plane_elems_all; };
    auto plane_elems = [&](int mp) { return MULTI && !mp ? s.ref_elems : plane_elems_all; };
    if (s.persist) {
        // Streaming blocks: every tile is a whole, vectorisable NCHW tile (host check).  A block walks tiles lin, lin + stride, ...
        // and issues the loads of its NEXT tile before it stores the current one, so HBM reads stay in flight for the whole launch
        // (one tile per block left the memory system idle while each block converted and stored).
        const int nt = ref_tiles + src_tiles, stride = s.persist;
        int cur = lin - wblocks;
        if (cur >= nt) return;
        auto decode = [&](int l, int &mp, int &nn, int &c0n, int &p0n) {
            mp = split_tile(l);
            nn = l / (tiles_p * tiles_c);
            const int rem = l - nn * (tiles_p * tiles_c);
            const int ct = rem / tiles_p;
            c0n = ct * TC; p0n = (rem - ct * tiles_p) * TPX;
        };
        float4 v[RPASS];
        int mp, nn, c0n, p0n;
        decode(cur, mp, nn, c0n, p0n);
        fast_load((mp ? s.src : s.ref) + (int64_t)nn * (mp ? s.src_stride[0] : s.ref_stride[0]), mp ? s.src_stride[1] : s.ref_stride[1], c0n, p0n, v);
        while (true) {
            fast_split(v);
            __syncthreads();
            const int nxt = cur + stride;
            int mp2 = 0, nn2 = 0, c02 = 0, p02 = 0;
            if (nxt < nt) {
                decode(nxt, mp2, nn2, c02, p02);
                fast_load((mp2 ? s.src : s.ref) + (int64_t)nn2 * (mp2 ? s.src_stride[0] : s.ref_stride[0]), mp2 ? s.src_stride[1] : s.ref_stride[1], c02, p02, v);
            }
            __nv_bfloat16 *hin = plane_hi(mp);
            fast_store(hin, hin + plane_elems(mp), nn, c0n, p0n);
            if (nxt >= nt) return;
            __syncthreads();
            cur = nxt; mp = mp2; nn = nn2; c0n = c02; p0n = p02;
        }
    }
    // reference and source tiles alternate in block order: when the source map is a peer-mapped tensor of another GPU its
    // NVLink reads (~0.77 TB/s, microsecond latency) overlap the local reference tiles instead of queueing behind them
    int map = 0;
    if (s.do_ref && s.do_src) map = split_tile(lin);
    else map = s.do_src ? 1 : 0;
    const int n = lin / (tiles_p * tiles_c), rem = lin % (tiles_p * tiles_c);
    const int c0 = (rem / tiles_p) * TC, p0 = (rem % tiles_p) * TPX;
    const T *base = map ? s.src : s.ref;
    const int64_t *strd = map ? s.src_stride : s.ref_stride;
    const int64_t sn = strd[0], sc = strd[1], sh = strd[2], sw = strd[3];
    const T *sp = base + (int64_t)n * sn;
    __nv_bfloat16 *hi = plane_hi(map), *lo = hi + plane_elems(map);
    const bool vec = nchw_vec4(sp, sc, sh, sw, W, HW);
    if (vec && sc != 1 && p0 + TPX <= HW && c0 + TC <= C) {
        float4 v[RPASS];
        fast_load(sp, sc, c0, p0, v);
        fast_split(v);
        __syncthreads();
        fast_store(hi, lo, n, c0, p0);
        return;
    }
    static_assert(NT == 256 && TC == 64 && TPX == 64 && TPITCH == 65, "stage_planes_tile's block and tile");
    stage_planes_tile<T, LO>(tile, sp, sc, sh, sw, vec, hi, lo, n, c0, p0, C, H, W);
}

template <typename T, typename... Tab>
static cudaError_t launch_stage_t(const T *ref, const int64_t ref_stride[4], const T *src, const int64_t src_stride[4],
                                  __nv_bfloat16 *planes, const float *P_ref, const float *P_src, PairGeom *pair_geom, uint16_t *order,
                                  float *order_key, const float *Wf, __nv_bfloat16 *w_planes, int w_add_identity, int *zero_words, int N,
                                  int n_ref, int n_views, int C, int H, int W, const GeomCfg &gc, cudaStream_t st, int &launched,
                                  const Tab &... vs) {
    StageArgs<T> s;
    s.ref = ref; s.src = src;
    for (int i = 0; i < 4; i++) { s.ref_stride[i] = ref_stride[i]; s.src_stride[i] = src_stride[i]; }
    s.planes = planes; s.P_ref = P_ref; s.P_src = P_src; s.pair_geom = pair_geom; s.order = order; s.order_key = order_key; s.Wf = Wf; s.w_planes = w_planes; s.w_add_identity = w_add_identity;
    s.zero_words = zero_words; s.N = N; s.n_ref = n_ref; s.n_views = n_views; s.C = C; s.H = H; s.W = W; s.gc = gc;
    s.do_ref = 1; s.do_src = n_views ? 0 : 1; s.do_order = (P_ref && P_src && order) ? 1 : 0; s.persist = 0;
    const int tiles_pc = ((H * W + stg::TPX - 1) / stg::TPX) * ((C + stg::TC - 1) / stg::TC);
    const int ref_items = n_views ? n_views * n_ref : n_ref;
    const int tiles = tiles_pc * ref_items + (n_views ? 0 : tiles_pc * N);   // reference tiles + source tiles
    s.ref_tiles = tiles_pc * ref_items;
    s.ref_elems = (size_t)ref_items * H * W * C;
    s.src_plane0 = (std::is_same<T, __nv_bfloat16>::value ? 1 : 2) * s.ref_elems;
    const int wblocks = (Wf && w_planes) ? (C * C / 8 + stg::NT - 1) / stg::NT : 0;        // C % 8 == 0
    // dynamic shared memory: the transposition tile, or (order blocks) 16 KB histogram + 2 B per pixel
    const size_t smem_tile = (size_t)stg::TC * stg::TPITCH * sizeof(float);
    const size_t smem_order = (size_t)stg::NBIN * 4 + (size_t)H * W * 2;
    const bool multi = n_ref != N || n_views;
    void (*kern)(const StageArgs<T>, const Tab...) = multi ? epi_stage_kernel<T, true, Tab...> : epi_stage_kernel<T, false, Tab...>;
    static thread_local size_t smem_set[kMaxDevices][2] = {};           // per device: the attribute applies to the current one
    const int dev = current_device();
    size_t uncached[2] = {0, 0};
    size_t *set = dev < kMaxDevices ? smem_set[dev] : uncached;
    auto ensure = [&](size_t smem) -> cudaError_t {
        if (smem + 1024 > 48 * 1024 && smem > set[multi]) {             // (+ the kernel's small static arrays)
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            set[multi] = smem;
        }
        return cudaSuccess;
    };
    // Shared memory is a per-launch size: above 64 KB the order blocks' pixel list would cut the residency of every transposition
    // block of the same launch, so maps that large order their pixels in a launch of their own (a no-op on a cached camera pair).
    const bool order_apart = s.do_order && smem_order > 64 * 1024;
    launched = order_apart ? 2 : 1;
    if (order_apart) {
        StageArgs<T> o = s;
        o.do_ref = 0; o.do_src = 0; o.Wf = nullptr; o.w_planes = nullptr; o.persist = 0;
        cudaError_t e = ensure(smem_order);
        if (e != cudaSuccess) return e;
        e = launch_pdl(kern, dim3((unsigned)N), dim3(stg::NT), smem_order, st, o, vs...);
        if (e != cudaSuccess) return e;
        s.do_order = 0; s.zero_words = nullptr;                  // the order launch has zeroed the counters
    }
    // streaming blocks when every tile of both maps is a whole, 16-byte-vectorisable NCHW tile
    auto whole = [&](const T *b, const int64_t *sd) {
        return sd[3] == 1 && sd[2] == W && sd[1] % 4 == 0 && sd[0] % 4 == 0 && sd[1] != 1 && (reinterpret_cast<uintptr_t>(b) & (4 * sizeof(T) - 1)) == 0;
    };
    s.persist = 0;
    if ((H * W) % stg::TPX == 0 && C % stg::TC == 0 && whole(ref, ref_stride) && (n_views || whole(src, src_stride))) {
        const int slots = 5 * sm_count();                      // 5 resident blocks per SM (__launch_bounds__)
        s.persist = tiles < slots ? tiles : slots;
    }
    const int grid = (s.do_order ? N : 0) + wblocks + (s.persist ? s.persist : tiles);
    const size_t smem = (s.do_order && smem_order > smem_tile) ? smem_order : smem_tile;
    cudaError_t e = ensure(smem);
    if (e != cudaSuccess) return e;
    return launch_pdl(kern, dim3((unsigned)grid), dim3(stg::NT), smem, st, s, vs...);
}

template <typename... Tab>
static cudaError_t launch_stage_d(const void *ref, const int64_t ref_stride[4], const void *src, const int64_t src_stride[4], int dtype,
                                  __nv_bfloat16 *planes, const float *P_ref, const float *P_src, PairGeom *pair_geom, uint16_t *order,
                                  float *order_key, const float *Wf, __nv_bfloat16 *w_planes, int w_add_identity, int *zero_words, int N,
                                  int n_ref, int n_views, int C, int H, int W, const GeomCfg &gc, cudaStream_t st, int &launched,
                                  const Tab &... vs) {
    if (dtype == kBF16)
        return launch_stage_t(static_cast<const __nv_bfloat16 *>(ref), ref_stride, static_cast<const __nv_bfloat16 *>(src), src_stride, planes,
                              P_ref, P_src, pair_geom, order, order_key, Wf, w_planes, w_add_identity, zero_words, N, n_ref, n_views, C, H, W, gc, st, launched, vs...);
    if (dtype == kF16)
        return launch_stage_t(static_cast<const __half *>(ref), ref_stride, static_cast<const __half *>(src), src_stride, planes,
                              P_ref, P_src, pair_geom, order, order_key, Wf, w_planes, w_add_identity, zero_words, N, n_ref, n_views, C, H, W, gc, st, launched, vs...);
    return launch_stage_t(static_cast<const float *>(ref), ref_stride, static_cast<const float *>(src), src_stride, planes,
                          P_ref, P_src, pair_geom, order, order_key, Wf, w_planes, w_add_identity, zero_words, N, n_ref, n_views, C, H, W, gc, st, launched, vs...);
}

cudaError_t launch_stage(const void *ref, const int64_t ref_stride[4], const void *src, const int64_t src_stride[4], int dtype,
                         __nv_bfloat16 *planes, const float *P_ref, const float *P_src, PairGeom *pair_geom, uint16_t *order,
                         float *order_key, const float *Wf, __nv_bfloat16 *w_planes, int w_add_identity, int *zero_words, int N, int n_ref,
                         int n_views, const ViewSources &vs, int C, int H, int W, const GeomCfg &gc, cudaStream_t st, int &launched) {
    if (vs.S)
        return launch_stage_d(ref, ref_stride, src, src_stride, dtype, planes, P_ref, P_src, pair_geom, order, order_key, Wf, w_planes,
                              w_add_identity, zero_words, N, n_ref, n_views, C, H, W, gc, st, launched, vs);
    return launch_stage_d(ref, ref_stride, src, src_stride, dtype, planes, P_ref, P_src, pair_geom, order, order_key, Wf, w_planes,
                          w_add_identity, zero_words, N, n_ref, n_views, C, H, W, gc, st, launched);
}

}  // namespace epi
