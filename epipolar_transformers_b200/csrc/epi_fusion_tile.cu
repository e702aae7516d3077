// epi_fusion_tile.cu — tensor-core fused kernel (warpgroup MMA), one CTA per 4x8 tile of reference pixels.
//
// Same arithmetic as the warp kernel (epi_fusion_warp.cu) but restructured around the linearity of
// bilinear sampling:      sim_k = Σ_t w_kt · (q · f[p_t])        out = Σ_p β_p · f[p],  β_p = Σ_{k,t→p} a_k w_kt
// so the per-pixel work becomes two dense GEMMs over the UNION of source pixels the tile's epipolar
// lines touch (D rows, gathered once per GEMM into shared memory):
//   GEMM1  S[d, i]  = Σ_c F[d, c] · Q[i, c]        (M = 128 source pixels / chunk, N = 32 ref pixels, K = C)
//   GEMM2  O[c, i]  = Σ_d F[d, c] · β[i, d]        (M = 128 channels,             N = 32 ref pixels, K = D)
// Operands are bf16 (hi, lo) pairs, three MMAs per product (hi·hi + hi·lo + lo·hi, fp32 accumulate in registers):
// ~2^-16 relative, inside the 1e-4 parity bar, where a single bf16/TF32 pass is not.  The gathered chunk
// F[d][c] sits in 128B-swizzled panels and is the K-major A operand of GEMM1 and — the same bytes read
// transposed — the MN-major A operand of GEMM2.  Between the GEMMs the CUDA cores interpolate the scores
// (4 taps per sample), run the softmax over K with warp shuffles, emit attn / corr_pos, and scatter the
// tap weights into β with deterministic fixed-point shared-memory atomics.
//
// Reference lines restated: /root/reference/modeling/layers/epipolar.py:199,210 (grid_sample taps),
// :295-307 (similarity, ==0 mask, scale, softmax), :237-243 (argmax, weighted sum), :323-418 (geometry).
#include <cuda_bf16.h>

#include "epi_kernels.cuh"
#include "epi_umma.cuh"

namespace epi {
using namespace umma;

namespace tile {
constexpr int TW = 8, TH = 4;     // tile of reference pixels (x, y)
constexpr int TM = TW * TH;       // = 32 = MMA N
constexpr int CHUNK = 128;        // union rows per MMA (M of GEMM1, K of GEMM2)
constexpr int DMAX = 480;         // max union size handled in one pass (table row length)
constexpr int NT = 512;           // worker threads
constexpr int NWARP = NT / 32;
constexpr int MAXWORDS = 512;     // bitmap words: H*W <= 16384
constexpr int MAXKPL = 4;         // samples per lane: K <= 128
constexpr float FIX = 1073741824.0f;   // 2^30 fixed point for the β scatter

constexpr uint32_t STAGE_BYTES = 65536;        // [hi: 2 panels x 16 KB][lo: 2 panels x 16 KB]
constexpr uint32_t PANEL_A = 16384;            // 128 rows x 128 B
constexpr uint32_t OFF_STAGE = 0;
constexpr uint32_t OFF_QB = 2 * STAGE_BYTES;                       // 32 KB: Q hi/lo panels | β chunk double buffer | attn tile
constexpr uint32_t OFF_TABLE = OFF_QB + 32768;                     // [32][DMAX] fp32 / int32
constexpr uint32_t OFF_BITMAP = OFF_TABLE + TM * DMAX * 4;
constexpr uint32_t OFF_PREFIX = OFF_BITMAP + MAXWORDS * 4;
constexpr uint32_t OFF_IDX = OFF_PREFIX + MAXWORDS * 4;
constexpr uint32_t OFF_ENDS = OFF_IDX + 512 * 2;
constexpr uint32_t OFF_MISC = OFF_ENDS + TM * 16;
constexpr uint32_t SMEM_BYTES = OFF_MISC + 512;
constexpr uint32_t SMEM_ALLOC = SMEM_BYTES + 1024;                 // 1024-byte alignment slack

constexpr uint32_t PANEL_B2 = 8192;  // stacked B panel: 64 rows x 128 B (rows 0-31 hi, 32-63 lo)

struct Misc {
    int stack[16];
    int sp;
    int total;
    int next_tile;
    int warp_tot[NWARP];
    PairGeom geom;
    uint16_t tpy[TM], tpx[TM];      // sector tiles: (y, x) of the tile's pixels, 0xFFFF = no pixel
};
static_assert(sizeof(Misc) <= 512, "Misc too large");

}  // namespace tile

using namespace tile;

#ifdef EPI_TILE_TIMERS
__device__ unsigned long long g_tile_timers[16];
#define TMARK(slot) do { if (tid == 0) { long long _t = clock64(); atomicAdd(&g_tile_timers[slot], (unsigned long long)(_t - t_prev)); t_prev = _t; } } while (0)
#else
#define TMARK(slot) do { } while (0)
#endif

template <int KPL, bool SECTOR>
__global__ void __launch_bounds__(NT, 1) epi_fusion_tile_kernel(const FusionArgs a, const ViewSources vs) {
    extern __shared__ uint8_t smem_raw[];
    // keep the shared address space visible to the compiler: offset arithmetic on the array, no integer casts
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *qb = smem + OFF_QB;
    float *table = reinterpret_cast<float *>(smem + OFF_TABLE);
    uint32_t *bitmap = reinterpret_cast<uint32_t *>(smem + OFF_BITMAP);
    uint32_t *prefix = reinterpret_cast<uint32_t *>(smem + OFF_PREFIX);
    uint16_t *idx = reinterpret_cast<uint16_t *>(smem + OFF_IDX);
    float4 *ends = reinterpret_cast<float4 *>(smem + OFF_ENDS);
    Misc &ms = *reinterpret_cast<Misc *>(smem + OFF_MISC);

    const int C = a.C, K = a.geom.K, H = a.geom.H, W = a.geom.W, HW = H * W;
    const int tiles_x = (W + TW - 1) / TW, tiles_y = (H + TH - 1) / TH;
    const int tiles_per_item = SECTOR ? (HW + TM - 1) / TM : tiles_x * tiles_y;
    const int total_tiles = a.N * tiles_per_item;
    int n = 0, ty0 = 0, tx0 = 0;                    // current tile (persistent CTA, dynamic tile scheduler)
    PairItems items = {0, 0};                       // its pair's query and source items
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wg = warp >> 2, t128 = tid & 127;     // warpgroup (MMA issue unit), thread within it
    const int nwords = (HW + 31) >> 5;
    const int NH = (C + 127) >> 7;                  // channel halves of 128
    const GeomCfg gc = a.geom;
    const float sl2 = a.softmax_scale * 1.4426950408889634f;
    const __nv_bfloat16 *src_hi = a.src_hi, *src_lo = a.src_lo;
    // tile pixel i -> (y, x), flattened index, validity
    // SECTOR: the tile is 32 consecutive entries of the per-pair list of pixels sorted by epipolar angle (their
    // epipolar lines nearly coincide, so the union of taps is ~2.4x smaller than for a 4x8 block); else a 4x8 block.
    auto pix_y = [&](int i) { return SECTOR ? (int)ms.tpy[i] : ty0 + (i >> 3); };
    auto pix_x = [&](int i) { return SECTOR ? (int)ms.tpx[i] : tx0 + (i & 7); };
    auto pix_ok = [&](int i) { return SECTOR ? ms.tpy[i] != 0xFFFFu : (ty0 + (i >> 3) < H && tx0 + (i & 7) < W); };

    int cur_n = -1;
#ifdef EPI_TILE_TIMERS
    long long t_prev = clock64();
#endif

  for (int tile = blockIdx.x; tile < total_tiles;) {
    {
        n = tile / tiles_per_item;
        const int trem = tile % tiles_per_item;
        if (SECTOR) {
            if (tid < TM) {
                const int e = trem * TM + tid;
                const unsigned p = e < HW ? a.order[(size_t)n * HW + e] : 0xFFFFu;
                ms.tpy[tid] = p == 0xFFFFu ? (uint16_t)0xFFFFu : (uint16_t)(p / W);
                ms.tpx[tid] = (uint16_t)(p == 0xFFFFu ? 0u : p % W);
            }
        } else {
            ty0 = (trem / tiles_x) * TH; tx0 = (trem % tiles_x) * TW;
        }
        items = pair_items(n, a.n_ref, a.n_views, vs);
        src_hi = a.src_hi + (size_t)items.s * HW * C; src_lo = a.src_lo + (size_t)items.s * HW * C;
    }
    if (tid == 32) {
        ms.sp = 1; ms.stack[0] = 0 | (TM << 8);
        if (!a.locs_in && n != cur_n) pair_geom_from_krt(a.P_ref + 12 * items.q, a.P_src + 12 * items.s, ms.geom);
    }
    if (tid == 64)      // claim the next tile now; its index is consumed after this tile (hides the atomic's latency)
        ms.next_tile = a.tile_counter ? (int)gridDim.x + atomicAdd(a.tile_counter, 1) : tile + (int)gridDim.x;
    cur_n = n;
    __syncthreads();
    if (tid < TM) {
        float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
        if (pix_ok(tid) && !a.locs_in)
            line_endpoints(ms.geom, gc, pix2coord(pix_x(tid), gc.ds, gc.r), pix2coord(pix_y(tid), gc.ds, gc.r), e.x, e.y, e.z, e.w);
        ends[tid] = e;
    }
    __syncthreads();

    // sample k of tile pixel i: normalised location (fused geometry or injected locations)
    auto sample_loc = [&](int i, int k, float &gx, float &gy) {
        if (a.locs_in) {
            const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + pix_y(i) * W + pix_x(i));
            gx = l.x; gy = l.y;
        } else {
            const float4 e = ends[i];
            const float t = (float)k / (float)(K - 1);
            gx = img2grid_x(e.x + (e.z - e.x) * t, gc);
            gy = img2grid_y(e.y + (e.w - e.y) * t, gc);
        }
    };
    auto rank_of = [&](int pix) { return (int)(prefix[pix >> 5] + __popc(bitmap[pix >> 5] & ((1u << (pix & 31)) - 1u))); };

    // ---------------- groups of pixels whose union of taps fits DMAX ----------------
    while (true) {
        __syncthreads();
        if (ms.sp == 0) break;
        const int top = ms.stack[ms.sp - 1];
        const int g0 = top & 0xff, gn = top >> 8;
        __syncthreads();
        if (tid == 0) ms.sp--;
        if (tid < nwords) bitmap[tid] = 0u;
        __syncthreads();
        // mark every in-bounds tap of every sample of the group's pixels.  lane <-> pixel, warp <-> sample
        // (k = warp, warp+16, ...): the 32 lanes of one atomic belong to 32 different epipolar lines, so they
        // spread over several bitmap words instead of piling onto the one word a single line crosses.
        {
            const int i = lane;
            if (i >= g0 && i < g0 + gn && pix_ok(i)) {
                for (int k = warp; k < K; k += NWARP) {
                    float gx, gy;
                    sample_loc(i, k, gx, gy);
                    const Taps t = make_taps(gx, gy, H, W, gc.align);
                    if (t.any) {
#pragma unroll
                        for (int tp = 0; tp < 4; tp++)
                            if (t.w[tp] != 0.f) {
                                const int pix = (t.y0 + (tp >> 1)) * W + t.x0 + (tp & 1);
                                atomicOr(&bitmap[pix >> 5], 1u << (pix & 31));
                            }
                    }
                }
            }
        }
        __syncthreads();
        // exclusive prefix of popcounts (one word per thread), total = D
        {
            const int v = tid < nwords ? __popc(bitmap[tid]) : 0;
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
            if (lane == 31) ms.warp_tot[warp] = incl;
            __syncthreads();
            int base = 0;
            for (int w = 0; w < warp; w++) base += ms.warp_tot[w];
            if (tid < nwords) prefix[tid] = base + incl - v;
            if (tid == NT - 1) ms.total = base + incl;
        }
        __syncthreads();
        const int D = ms.total;
        TMARK(0);
        if (D > DMAX) {                       // split the group (a single pixel always fits: launch-time check)
            if (gn <= 1) __trap();
            if (tid == 0) {
                const int h1 = gn >> 1;
                ms.stack[ms.sp++] = (g0 + h1) | ((gn - h1) << 8);
                ms.stack[ms.sp++] = g0 | (h1 << 8);
            }
            continue;
        }
        // union list: idx[rank] = source pixel
        if (tid < nwords) {
            uint32_t bits = bitmap[tid];
            int r = prefix[tid];
            while (bits) { const int b = __ffs(bits) - 1; bits &= bits - 1; idx[r++] = (uint16_t)(tid * 32 + b); }
        }
        const int nch = (D + CHUNK - 1) / CHUNK;

        // ---------------- Q operand: [32 px][C] -> bf16 (hi, lo) K-major panels ----------------
        if (SECTOR) {
            // the reference map was split to bf16 planes [HW][C] by the staging kernel: 16-byte chunk copies
            const int C8 = C >> 3, J = NH * 16, jsh = NH == 1 ? 4 : 5;      // J is 16 or 32
            for (int e = tid; e < 2 * TM * J; e += NT) {
                    const int plane = e >> (jsh + 5), rem = e & ((TM << jsh) - 1), i = rem >> jsh, j = rem & (J - 1);
                    uint4 v = make_uint4(0u, 0u, 0u, 0u);
                    if (i >= g0 && i < g0 + gn && pix_ok(i) && j < C8)
                        v = __ldg(reinterpret_cast<const uint4 *>((plane ? a.ref_lo : a.ref_hi) +
                                                                  ((size_t)items.q * HW + pix_y(i) * W + pix_x(i)) * C + j * 8));
                    *reinterpret_cast<uint4 *>(qb + (j >> 3) * PANEL_B2 + plane * 4096u + i * 128u + (((j & 7) ^ (i & 7)) << 4)) = v;
                }
        } else
        {
            const int i = lane;
            const bool ok = i >= g0 && i < g0 + gn && pix_ok(i);
            const float *rb = a.feat_ref + (int64_t)items.q * a.ref_stride[0] + (int64_t)pix_y(i) * a.ref_stride[2] + (int64_t)pix_x(i) * a.ref_stride[3];
            const int64_t sc = a.ref_stride[1];
            {
                float f[2][8];
#pragma unroll
                for (int it = 0; it < 2; it++) {                   // groups of 8 channels: cg = warp, warp + 16
                    const int cg = warp + it * NWARP;
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int c = cg * 8 + u;
                        f[it][u] = (ok && cg < NH * 16 && c < C) ? __ldg(rb + c * sc) : 0.f;
                    }
                }
#pragma unroll
                for (int it = 0; it < 2; it++) {
                    const int cg = warp + it * NWARP;
                    if (cg < NH * 16) {
                        uint4 hi, lo;
                        split8(f[it], hi, lo);
                        const uint32_t off = (cg >> 3) * PANEL_B2 + i * 128u + (((cg & 7) ^ (i & 7)) << 4);
                        *reinterpret_cast<uint4 *>(qb + off) = hi;
                        *reinterpret_cast<uint4 *>(qb + 4096 + off) = lo;
                    }
                }
            }
        }
        __syncthreads();      // idx + Q visible
        TMARK(1);

        // gather of one stage: rows idx[c*128 .. +127], channels [128h, 128h+128) of both planes (16-byte chunks).
        // Split into load (global -> registers) and store (registers -> swizzled panels) so the loads of stage
        // s+1 are in flight while stage s is fenced, synchronised and handed to the tensor core.
        const int g_sub = lane >> 4, g_j = lane & 15;              // 16 lanes x 16 B = one 256-byte row half
        auto gather_load = [&](uint4 (&v)[8], int c, int h) {
            const int ch0 = h * 128 + g_j * 8;
#pragma unroll
            for (int it = 0; it < 8; it++) {
                const int plane = it >> 2;
                const int r = (it & 3) * 32 + warp * 2 + g_sub;
                const int d = c * CHUNK + r;
                v[it] = make_uint4(0u, 0u, 0u, 0u);
                if (d < D && ch0 < C) {
                    const __nv_bfloat16 *row = (plane ? src_lo : src_hi) + (size_t)idx[d] * C + ch0;
                    v[it] = __ldg(reinterpret_cast<const uint4 *>(row));
                }
            }
        };
        auto gather_store = [&](uint8_t *stage, const uint4 (&v)[8]) {
#pragma unroll
            for (int it = 0; it < 8; it++) {
                const int plane = it >> 2;
                const int r = (it & 3) * 32 + warp * 2 + g_sub;
                const uint32_t off = plane * 32768u + (g_j >> 3) * PANEL_A + r * 128u + (((g_j & 7) ^ (r & 7)) << 4);
                *reinterpret_cast<uint4 *>(stage + off) = v[it];
            }
        };
        // Stage st is double-buffered (buffer st & 1) and consumed synchronously: every warpgroup waits for its MMAs on stage st
        // before the barrier of stage st + 1, so the buffer is free again when stage st + 2 is stored.
        const int n_st = nch * NH;

        // ---------------- phase A: S = F·Qᵀ -> table[i][d] ----------------
        // Warpgroup wg accumulates union rows c * 128 + (wg & 1) * 64 .. +63 of the chunks c with c % 2 == wg >> 1.
        {
            float sacc[2][16];
#pragma unroll
            for (int e = 0; e < 16; e++) { sacc[0][e] = 0.f; sacc[1][e] = 0.f; }
            uint4 v[8];
            if (n_st > 0) gather_load(v, 0, 0);
            for (int st = 0; st < n_st; st++) {
                const int c = st / NH, h = st % NH;
                uint8_t *stage = smem + OFF_STAGE + (st & 1) * STAGE_BYTES;
                gather_store(stage, v);
                if (st + 1 < n_st) gather_load(v, (st + 1) / NH, (st + 1) % NH);
                fence_proxy_async_smem();
                __syncthreads();                                    // stage st is in shared memory
                if ((c & 1) == (wg >> 1) && c * CHUNK + (wg & 1) * 64 < D) {
                    const uint32_t sa = smem_u32(stage) + (uint32_t)(wg & 1) * 8192u, sq = smem_u32(qb);
                    wg_fence();
#pragma unroll
                    for (int ks = 0; ks < 8; ks++) {
                        const uint32_t ao = (ks >> 2) * PANEL_A + (ks & 3) * 32, bo = (h * 2 + (ks >> 2)) * PANEL_B2 + (ks & 3) * 32;
                        const uint64_t a_hi = make_smem_desc(sa + ao, 16, 1024), a_lo = desc_add(a_hi, 32768);
                        const uint64_t b = make_smem_desc(sq + bo, 16, 1024), b_lo = desc_add(b, 4096);
                        if (c >> 1) { wgmma_m64n32<0>(sacc[1], a_hi, b); wgmma_m64n32<0>(sacc[1], a_hi, b_lo); wgmma_m64n32<0>(sacc[1], a_lo, b); }
                        else        { wgmma_m64n32<0>(sacc[0], a_hi, b); wgmma_m64n32<0>(sacc[0], a_hi, b_lo); wgmma_m64n32<0>(sacc[0], a_lo, b); }
                    }
                    wg_commit();
                    wg_wait_all();
                }
            }
            TMARK(2);
#pragma unroll
            for (int q = 0; q < 2; q++) {
                const int c = 2 * q + (wg >> 1);
                if (c < nch) {
#pragma unroll
                    for (int e = 0; e < 16; e++) {
                        const int d = c * CHUNK + (wg & 1) * 64 + acc_row(t128, e);
                        if (d < D) table[acc_col(t128, e) * DMAX + d] = sacc[q][e];
                    }
                }
            }
        }
        __syncthreads();

        TMARK(3);
        // ---------------- phase B2: interpolate scores, softmax over K, outputs, β scatter ----------------
        float *attn_tile = reinterpret_cast<float *>(qb);         // [K][32]; Q panels are dead now
        {
            // Each warp owns up to two pixels (i0, i0+16) and runs them interleaved for instruction-level
            // parallelism; lane <-> sample.  Tap ranks and weights are kept in registers for the β scatter.
            constexpr int PW = TM / NWARP;                         // 2
            float x[PW][KPL], gxs[PW][KPL], gys[PW][KPL], tw[PW][KPL][4];
            uint32_t rk[PW][KPL][2];                            // 4 ranks, packed 2 x u16
            bool act[PW];
            float mx[PW];
#pragma unroll
            for (int u = 0; u < PW; u++) {
                const int i = g0 + warp + u * NWARP;
                act[u] = i < g0 + gn && pix_ok(i);
                mx[u] = -INFINITY;
#pragma unroll
                for (int j = 0; j < KPL; j++) {
                    const int k = j * 32 + lane;
                    x[u][j] = -INFINITY; gxs[u][j] = 0.f; gys[u][j] = 0.f; rk[u][j][0] = rk[u][j][1] = 0u;
#pragma unroll
                    for (int tp = 0; tp < 4; tp++) tw[u][j][tp] = 0.f;
                    if (act[u] && k < K) {
                        float gx, gy;
                        sample_loc(i, k, gx, gy);
                        gxs[u][j] = gx; gys[u][j] = gy;
                        if (a.locs_out)
                            reinterpret_cast<float2 *>(a.locs_out)[((size_t)k * a.N + n) * HW + pix_y(i) * W + pix_x(i)] = make_float2(gx, gy);
                        const Taps t = make_taps(gx, gy, H, W, gc.align);
                        float sim = 0.f;
                        if (t.any) {
                            uint32_t r[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                            for (int tp = 0; tp < 4; tp++)
                                if (t.w[tp] != 0.f) {
                                    r[tp] = (uint32_t)rank_of((t.y0 + (tp >> 1)) * W + t.x0 + (tp & 1));
                                    tw[u][j][tp] = t.w[tp];
                                    sim = fmaf(t.w[tp], table[i * DMAX + r[tp]], sim);
                                }
                            rk[u][j][0] = r[0] | (r[1] << 16); rk[u][j][1] = r[2] | (r[3] << 16);
                        }
                        if (sim == 0.f) sim = kMasked;                      // epipolar.py:298
                        x[u][j] = sim * sl2;
                        mx[u] = fmaxf(mx[u], x[u][j]);
                    }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                for (int u = 0; u < PW; u++) mx[u] = fmaxf(mx[u], __shfl_xor_sync(0xffffffffu, mx[u], o));
            float sum[PW];
#pragma unroll
            for (int u = 0; u < PW; u++) {
                sum[u] = 0.f;
#pragma unroll
                for (int j = 0; j < KPL; j++) { x[u][j] = (act[u] && j * 32 + lane < K) ? exp2f(x[u][j] - mx[u]) : 0.f; sum[u] += x[u][j]; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                for (int u = 0; u < PW; u++) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
#pragma unroll
            for (int u = 0; u < PW; u++) {
                if (!act[u]) continue;                              // warp-uniform
                const int i = g0 + warp + u * NWARP;
                const float inv = 1.f / sum[u];
                float best_v = -1.f, best_gx = 0.f, best_gy = 0.f;
                int best_k = 0x7fffffff;
#pragma unroll
                for (int j = 0; j < KPL; j++) {
                    const int k = j * 32 + lane;
                    x[u][j] *= inv;
                    if (k < K) {
                        if (a.attn) attn_tile[k * TM + i] = x[u][j];
                        if (x[u][j] > best_v) { best_v = x[u][j]; best_k = k; best_gx = gxs[u][j]; best_gy = gys[u][j]; }
                    }
                }
                if (a.corr_pos) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
                        const int ok = __shfl_xor_sync(0xffffffffu, best_k, o);
                        const float ogx = __shfl_xor_sync(0xffffffffu, best_gx, o), ogy = __shfl_xor_sync(0xffffffffu, best_gy, o);
                        if (EPI_FIRST_MAX_BEATS(ov, ok, best_v, best_k)) { best_v = ov; best_k = ok; best_gx = ogx; best_gy = ogy; }
                    }
                    if (lane == 0)
                        reinterpret_cast<float2 *>(a.corr_pos)[(size_t)n * HW + pix_y(i) * W + pix_x(i)] =
                            make_float2(grid2corr(best_gx, W, gc.correct), grid2corr(best_gy, H, gc.correct));
                }
                // β row: zero, then deterministic fixed-point scatter of a_k·w_kt
                int *trow = reinterpret_cast<int *>(table + i * DMAX);
                __syncwarp();
                for (int d = lane; d < D; d += 32) trow[d] = 0;
                __syncwarp();
#pragma unroll
                for (int j = 0; j < KPL; j++) {
                    if (j * 32 + lane < K) {
#pragma unroll
                        for (int tp = 0; tp < 4; tp++)
                            if (tw[u][j][tp] != 0.f) {
                                const uint32_t r = (rk[u][j][tp >> 1] >> ((tp & 1) * 16)) & 0xffffu;
                                atomicAdd(&trow[r], __float2int_rn(x[u][j] * tw[u][j][tp] * FIX));
                            }
                    }
                }
            }
        }
        __syncthreads();
        TMARK(4);
        if (a.attn) {       // flush the attention tile: 8-pixel row segments
            float *ab = a.attn + (size_t)n * K * HW;
            for (int e = tid; e < K * TM; e += NT) {
                const int i = e & 31, k = e >> 5;
                if (i >= g0 && i < g0 + gn && pix_ok(i)) ab[(size_t)k * HW + pix_y(i) * W + pix_x(i)] = attn_tile[k * TM + i];
            }
        }
        __syncthreads();

        TMARK(5);
        // ---------------- phase C: Oᵀ = Fᵀ·βᵀ ----------------
        // Warpgroup wg accumulates channels (wg >> 1) * 128 + (wg & 1) * 64 .. +63 over all chunks.
        float oacc[16];
#pragma unroll
        for (int e = 0; e < 16; e++) oacc[e] = 0.f;
        {
            uint4 v[8];
            if (n_st > 0) gather_load(v, 0, 0);
            for (int st = 0; st < n_st; st++) {
                const int c = st / NH, h = st % NH;
                uint8_t *bb = qb + (c & 1) * 16384;
                uint8_t *stage = smem + OFF_STAGE + (st & 1) * STAGE_BYTES;
                gather_store(stage, v);
                if (st + 1 < n_st) gather_load(v, (st + 1) / NH, (st + 1) % NH);
                if (h == 0) {
                    // β chunk -> bf16 (hi, lo) K-major panels [32 px][128 d]: thread <-> (pixel, 8 consecutive d)
                    const int i = tid >> 4, dg = tid & 15;
                    const bool ok = i >= g0 && i < g0 + gn;
                    float f[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int d = c * CHUNK + dg * 8 + u;
                        f[u] = (ok && d < D) ? (float)reinterpret_cast<const int *>(table)[i * DMAX + d] * (1.0f / FIX) : 0.f;
                    }
                    uint4 hi, lo;
                    split8(f, hi, lo);
                    const uint32_t off = (dg >> 3) * PANEL_B2 + i * 128u + (((dg & 7) ^ (i & 7)) << 4);
                    *reinterpret_cast<uint4 *>(bb + off) = hi;
                    *reinterpret_cast<uint4 *>(bb + 4096 + off) = lo;
                }
                fence_proxy_async_smem();
                __syncthreads();
                if (h == (wg >> 1)) {
                    const uint32_t sa = smem_u32(stage) + (uint32_t)(wg & 1) * PANEL_A, sb = smem_u32(bb);
                    wg_fence();
#pragma unroll
                    for (int ks = 0; ks < 8; ks++) {
                        const uint32_t ao = ks * 2048, bo = (ks >> 2) * PANEL_B2 + (ks & 3) * 32;
                        const uint64_t a_hi = make_smem_desc(sa + ao, PANEL_A, 1024), a_lo = desc_add(a_hi, 32768);
                        const uint64_t b = make_smem_desc(sb + bo, 16, 1024), b_lo = desc_add(b, 4096);
                        wgmma_m64n32<1>(oacc, a_hi, b); wgmma_m64n32<1>(oacc, a_hi, b_lo); wgmma_m64n32<1>(oacc, a_lo, b);
                    }
                    wg_commit();
                    wg_wait_all();
                }
            }
        }
        __syncthreads();                                            // every warpgroup's MMAs are done with the stages

        TMARK(6);
        // ---------------- phase D: fused feature registers -> shared (transposed) -> global ----------------
        {
            // o_tile[i][ch] in the (now idle) stage buffers; row stride 260 floats keeps float4 alignment
            float *o_tile = reinterpret_cast<float *>(smem + OFF_STAGE);
            constexpr int OS = 260;
            if ((wg >> 1) < NH) {
                const int cb = (wg >> 1) * 128 + (wg & 1) * 64;
#pragma unroll
                for (int e = 0; e < 16; e++) o_tile[acc_col(t128, e) * OS + cb + acc_row(t128, e)] = nch ? oacc[e] : 0.f;   // nch==0: every sample masked, zero vectors
            }
            __syncthreads();
            if (a.out_hi) {
                // bf16 (hi, lo) planes [N][HW][C]: the A operand of the z-projection GEMM; one 16-byte store per lane
                for (int i = g0 + warp; i < g0 + gn; i += NWARP) {
                    if (!pix_ok(i) || lane * 8 >= C) continue;
                    float f[8];
                    *reinterpret_cast<float4 *>(f) = *reinterpret_cast<const float4 *>(o_tile + i * OS + lane * 8);
                    *reinterpret_cast<float4 *>(f + 4) = *reinterpret_cast<const float4 *>(o_tile + i * OS + lane * 8 + 4);
                    uint4 hi, lo;
                    split8(f, hi, lo);
                    const size_t o = ((size_t)n * HW + pix_y(i) * W + pix_x(i)) * C + lane * 8;
                    *reinterpret_cast<uint4 *>(a.out_hi + o) = hi;
                    *reinterpret_cast<uint4 *>(a.out_lo + o) = lo;
                }
            } else if (a.out_stride[1] != 1) {
                // NCHW-like: lane <-> tile pixel, so a warp store covers 4 segments of 8 consecutive pixels
                const int i = lane;
                const bool ok = i >= g0 && i < g0 + gn && pix_ok(i);
                float *ob = a.out + (int64_t)n * a.out_stride[0] + (int64_t)pix_y(i) * a.out_stride[2] + (int64_t)pix_x(i) * a.out_stride[3];
                const float *rb = a.feat_ref + (int64_t)items.q * a.ref_stride[0] + (int64_t)pix_y(i) * a.ref_stride[2] + (int64_t)pix_x(i) * a.ref_stride[3];
                if (ok)
                    for (int ch = warp; ch < C; ch += NWARP) {
                        float o = o_tile[i * OS + ch];
                        if (a.add_ref) o += __ldg(rb + ch * a.ref_stride[1]);
                        ob[ch * a.out_stride[1]] = o;
                    }
            } else {
                // channels-last: lane <-> channel
                for (int i = g0 + warp; i < g0 + gn; i += NWARP) {
                    if (!pix_ok(i)) continue;
                    float *ob = a.out + (int64_t)n * a.out_stride[0] + (int64_t)pix_y(i) * a.out_stride[2] + (int64_t)pix_x(i) * a.out_stride[3];
                    const float *rb = a.feat_ref + (int64_t)items.q * a.ref_stride[0] + (int64_t)pix_y(i) * a.ref_stride[2] + (int64_t)pix_x(i) * a.ref_stride[3];
                    for (int ch = lane; ch < C; ch += 32) {
                        float o = o_tile[i * OS + ch];
                        if (a.add_ref) o += __ldg(rb + ch * a.ref_stride[1]);
                        ob[ch] = o;
                    }
                }
            }
        }
        TMARK(7);
#ifdef EPI_TILE_TIMERS
        if (tid == 0) atomicAdd(&g_tile_timers[8], 1ull);
#endif
    }
    // next tile: dynamic (atomic counter zeroed by the operand-staging kernel) or static round-robin
    __syncthreads();
    tile = ms.next_tile;
    __syncthreads();
  }
}

bool fusion_tile_shape_ok(int C, int H, int W, int K, bool has_locs_in) {
    if (C % 8 != 0 || C > 256) return false;
    if (H * W > MAXWORDS * 32 || H * W > 65535) return false;
    if (K > 32 * MAXKPL) return false;
    // a single pixel's union must fit DMAX: 4 taps per sample, and (fused geometry) a straight line
    // crosses at most H+W pixel rows/columns, 2 pixels wide, plus the footprint ends
    const int single = has_locs_in ? 4 * K : min(4 * K, 2 * (H + W) + 8);
    return single <= DMAX;
}

cudaError_t launch_fusion_tile(const FusionArgs &a, const ViewSources &vs, cudaStream_t st) {
    const bool sector = a.order != nullptr;
    const int HW = a.geom.H * a.geom.W;
    const int tiles = a.N * (sector ? (HW + TM - 1) / TM : ((a.geom.W + TW - 1) / TW) * ((a.geom.H + TH - 1) / TH));
    const int kpl = (a.geom.K + 31) / 32;
    void (*kern)(const FusionArgs, const ViewSources);
    if (sector) kern = kpl <= 1 ? epi_fusion_tile_kernel<1, true> : (kpl <= 2 ? epi_fusion_tile_kernel<2, true> : epi_fusion_tile_kernel<4, true>);
    else        kern = kpl <= 1 ? epi_fusion_tile_kernel<1, false> : (kpl <= 2 ? epi_fusion_tile_kernel<2, false> : epi_fusion_tile_kernel<4, false>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_ALLOC);
    if (e != cudaSuccess) return e;
    const int sms = sm_count();
    const int grid = a.tile_counter ? (tiles < sms ? tiles : sms) : tiles;     // one persistent CTA per SM
    kern<<<grid, NT, SMEM_ALLOC, st>>>(a, vs);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// Per-pair list of reference pixels sorted by the angle of (pixel - e1) around the epipole e1 = P_ref·C_src of the
// source camera in the reference view: pixels on one epipolar line of the reference view share one epipolar line
// in the source view, so consecutive list entries have nearly identical tap sets.  One CTA per pair, bitonic sort
// of (16-bit angle key << 14 | pixel index) in shared memory — unique keys, hence a deterministic order.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) sector_order_kernel(const float *__restrict__ P_ref, const float *__restrict__ P_src,
                                                            uint16_t *__restrict__ order, int n_ref, int n_views, const ViewSources vs,
                                                            const GeomCfg gc) {
    extern __shared__ uint32_t keys[];
    __shared__ float s_e[4];          // ex, ey, a0, parallel-flag
    const int n = blockIdx.x, HW = gc.H * gc.W, W = gc.W;
    int npad = 1;
    while (npad < HW) npad <<= 1;
    if (threadIdx.x == 0) {
        const PairItems items = pair_items(n, n_ref, n_views, vs);
        const float *P1 = P_ref + 12 * items.q, *P2 = P_src + 12 * items.s;
        double a[9], t1[3], b[9], t2[3], bi[9], cs[3], e[3];
        cam_load(P2, b, t2);
        cam_inverse(b, bi);
        cam_centre(bi, t2, cs);                     // source camera centre
        cam_load(P1, a, t1);
        for (int r = 0; r < 3; r++) e[r] = cam_project(a, t1, cs, r);
        const double cx = 0.5 * ((double)gc.xmin + gc.xmax), cy = 0.5 * ((double)gc.ymin + gc.ymax);
        const double nrm = fabs(e[0]) + fabs(e[1]) + 1e-300;
        if (!(fabs(e[2]) > 1e-9 * nrm)) {        // epipole at infinity (or NaN): lines are parallel to (e0, e1): sort by the offset across them
            s_e[0] = (float)(e[0] / nrm); s_e[1] = (float)(e[1] / nrm); s_e[2] = 0.f; s_e[3] = 1.f;
        } else {
            const double ex = e[0] / e[2], ey = e[1] / e[2];
            s_e[0] = (float)ex; s_e[1] = (float)ey; s_e[2] = (float)atan2(cy - ey, cx - ex); s_e[3] = 0.f;
        }
    }
    __syncthreads();
    const float ex = s_e[0], ey = s_e[1], a0 = s_e[2];
    const bool parallel = s_e[3] != 0.f;
    const float span = fabsf(gc.xmax - gc.xmin) + fabsf(gc.ymax - gc.ymin) + 1.f;
    for (int i = threadIdx.x; i < npad; i += blockDim.x) {
        uint32_t v = 0xFFFFFFFFu;
        if (i < HW) {
            const float px = pix2coord(i % W, gc.ds, gc.r), py = pix2coord(i / W, gc.ds, gc.r);
            float u;                                   // in [0, 1)
            if (parallel) {
                u = 0.5f + 0.5f * ((px - 0.5f * (gc.xmin + gc.xmax)) * (-ey) + (py - 0.5f * (gc.ymin + gc.ymax)) * ex) / span;
            } else {
                float ang = atan2f(py - ey, px - ex) - a0;         // relative to the image centre: the cut is behind the epipole
                if (ang < -3.14159265f) ang += 6.28318531f;
                if (ang >= 3.14159265f) ang -= 6.28318531f;
                u = (ang + 3.14159265f) * (1.f / 6.28318531f);
            }
            u = fminf(fmaxf(u, 0.f), 0.99999f);
            if (!(u == u)) u = 0.f;
            v = ((uint32_t)(u * 65536.f) << 14) | (uint32_t)i;
        }
        keys[i] = v;
    }
    __syncthreads();
    for (int k = 2; k <= npad; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < npad; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const uint32_t x = keys[i], y = keys[l];
                    const bool up = (i & k) == 0;
                    if ((x > y) == up) { keys[i] = y; keys[l] = x; }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < HW; i += blockDim.x) order[(size_t)n * HW + i] = (uint16_t)(keys[i] & 0x3FFFu);
}

cudaError_t launch_sector_order(const float *P_ref, const float *P_src, uint16_t *order, int N, int n_ref, int n_views,
                                const ViewSources &vs, const GeomCfg &gc, cudaStream_t st) {
    const int HW = gc.H * gc.W;
    int npad = 1;
    while (npad < HW) npad <<= 1;
    const size_t smem = (size_t)npad * 4;
    cudaError_t e = cudaFuncSetAttribute(sector_order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    sector_order_kernel<<<N, 1024, smem, st>>>(P_ref, P_src, order, n_ref, n_views, vs, gc);
    return cudaGetLastError();
}

#ifdef EPI_TILE_TIMERS
extern "C" void epi_tile_timers_read(unsigned long long *out16, int reset) {
    cudaMemcpyFromSymbol(out16, g_tile_timers, sizeof(unsigned long long) * 16);
    if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_tile_timers, z, sizeof(z)); }
}
#endif

}  // namespace epi
