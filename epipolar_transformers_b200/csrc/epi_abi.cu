// epi_abi.cu — the extern "C" boundary declared in include/epipolar_b200.h.
// Validates arguments, plans the forward (kernels, staging, workspace and cache regions) and launches the plan on the caller's stream.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/epipolar_b200.h"
#include "epi_kernels.cuh"

namespace {

thread_local char g_err[512] = "";
thread_local int g_launches = 0;
thread_local int g_timing = 0, g_timing_valid = 0;
thread_local int g_items32 = 0;          // epi_pipe_force_items32: test and A/B-timing hook, not part of the public API
thread_local cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr, g_evA = nullptr, g_evB = nullptr;   // A: call start, B: call end

int fail(int code, const char *fmt, const char *detail = "") {
    snprintf(g_err, sizeof(g_err), fmt, detail);
    return code;
}

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

constexpr size_t NONE = ~(size_t)0;      // offset of a region the plan does not use

template <typename T>
T *at(void *base, size_t off) { return off == NONE ? nullptr : reinterpret_cast<T *>(static_cast<char *>(base) + off); }

// Consecutive regions of one buffer, each starting on a 256-byte boundary.  part() places a buffer right behind the previous one
// in the same region (planes a kernel addresses from one base, such as [hi | lo]); close() ends the region.
struct Regions {
    size_t end = 0;
    size_t part(size_t bytes) { const size_t off = end; end += bytes; return off; }
    void close() { end = align_up(end); }
    size_t take(size_t bytes) { const size_t off = part(bytes); close(); return off; }
};

// Counts the kernels a call launches and turns a failed launch into EPI_ECUDA "<what> launch failed: <CUDA error>".
struct Launches {
    int n = 0;
    int operator()(const char *what, cudaError_t e, int kernels = 1) {
        if (e == cudaSuccess) { n += kernels; return EPI_OK; }
        snprintf(g_err, sizeof(g_err), "%s launch failed: %s", what, cudaGetErrorString(e));
        return EPI_ECUDA;
    }
};

// EpiFusionParams.feat_dtype: the maps' element type in bits 0-7, `out`'s in bits 8-15 (EPI_OUT_DTYPE; 0 = float32)
inline int map_dtype(const EpiFusionParams *p) { return p->feat_dtype & 0xff; }
inline int out_dtype(const EpiFusionParams *p) { return (p->feat_dtype >> 8) & 0xff; }
inline bool out_dtype_ok(const EpiFusionParams *p) { return (p->feat_dtype & ~0xffff) == 0 && out_dtype(p) <= EPI_DTYPE_F16; }

// source views per reference item (EpiFusionParams.n_src: 0 and 1 both mean one)
inline int n_sources(const EpiFusionParams *p) { return p->n_src > 1 ? p->n_src : 1; }
// The views form's source table: every other view (S = 0) for epi_fusion_forward_f32, the caller's table for the
// epi_fusion_view_sources_* entry points
static_assert(EPI_VIEW_SOURCES_MAX == epi::kMaxViewSources, "the header's table limit is the kernels' by-value table size");
const epi::ViewSources kAllOthers{};
// sources per view in the views form: the table's width, or V−1
inline int view_sources(const EpiFusionParams *p, const epi::ViewSources &vs) { return vs.S ? vs.S : p->n_views - 1; }
// (query, source) pairs = items of out, attn, corr_pos and the sample locations: S·N, or V·S·N in the views form
inline int64_t n_pairs64(const EpiFusionParams *p, const epi::ViewSources &vs) {
    return p->n_views ? (int64_t)p->n_views * view_sources(p, vs) * p->N : (int64_t)n_sources(p) * p->N;
}
inline int n_pairs(const EpiFusionParams *p, const epi::ViewSources &vs) { return (int)n_pairs64(p, vs); }
// The views form (n_views = V) has one map, feat_ref with its V·N view items, that is both the query and the source map.
inline int n_ref_items(const EpiFusionParams *p) { return p->n_views ? p->n_views * p->N : p->N; }
inline int n_src_items(const EpiFusionParams *p) { return p->n_views ? p->n_views * p->N : n_sources(p) * p->N; }
inline const void *src_map(const EpiFusionParams *p) { return p->n_views ? p->feat_ref : p->feat_src; }
inline const int64_t *src_strides(const EpiFusionParams *p) { return p->n_views ? p->ref_stride : p->src_stride; }

bool src_is_channels_last(const EpiFusionParams *p) {
    const int64_t *s = src_strides(p);
    const int64_t C = p->C, H = p->H, W = p->W;
    return s[1] == 1 && s[3] == C && s[2] == W * C && (n_src_items(p) == 1 || s[0] == H * W * C) &&
           (reinterpret_cast<uintptr_t>(src_map(p)) % 16 == 0);
}

enum class Kernel { Pipe, Sector, Tile, Warp };          // fused attention kernel (sector and 4x8 block tiles: epi_fusion_tile_kernel)
enum class Staging { Pipe, Planes, Nhwc, InPlace };      // feat_src: the pipe's staging launch, bf16 (hi, lo) planes, fp32 channels-last, as is
enum class RefCopy { None, Before, After };              // fp32 channels-last copy of a low-precision feat_ref, before / after the fused kernel
// who writes `out`: the fused kernel, a transposition pass, the z GEMM / z epilogue; Head: the head kernel writes the heat-maps
// (epi_fusion_heatmaps_f32 only) from the fused kernel's pixel-major plane
enum class Epilogue { Direct, Unstage, ZGemm, ZFp32, Head };

// Everything the forward decides, made from the params alone.  Offsets are NONE for the regions the plan does not use.
struct Plan {
    const char *refusal = nullptr;       // a forced variant this shape cannot run
    Kernel kernel = Kernel::Warp;
    Staging staging = Staging::InPlace;
    RefCopy ref_copy = RefCopy::None;
    Epilogue epilogue = Epilogue::Direct;
    bool cached = false;                 // pair constants, pixel order and work records live in the caller's persistent cache
    size_t ref_hi = NONE, ref_lo = NONE, src_hi = NONE, src_lo = NONE, src_nhwc = NONE, ref32 = NONE;      // workspace
    size_t fused = NONE, fused_lo = NONE, counter = NONE, w_hi = NONE, w_lo = NONE, workspace_bytes = 0;
    size_t order = NONE, geom = NONE;    // pixel order and pair constants: in the cache when `cached`, else in the workspace
    size_t key = NONE, records = NONE, cache_bytes = 0;     // cache: per pair a key of 32 words (word 31: epoch of its work records)
    int n_records = 0;
    int item_px = 32;                    // pipe kernel: reference pixels per work item
};

bool want_pipe(const EpiFusionParams *p) {
    if (p->variant != EPI_VARIANT_AUTO && p->variant != EPI_VARIANT_PIPE) return false;
    if (!epi::fusion_pipe_shape_ok(p->C, p->H, p->W, p->K, p->sample_locs_in != nullptr)) return false;
    // Automatic selection leaves one corner to the other kernels: K > 48 on maps of 2K pixels or more a side.  There a single pixel's
    // taps (4K, sampled sparsely along a long line) already fill the 256-row union, so every work item splits down to one pixel.
    // The tile kernel takes that corner where its shape limits allow (C <= 256, at most 16384 pixels), the warp kernel otherwise
    // (tools/gpu_mapsize.py times the kernels per map size).
    if (p->variant == EPI_VARIANT_AUTO && 4 * p->K > 192 && (p->H > p->W ? p->H : p->W) >= 2 * p->K) return false;
    return true;
}

bool want_tile(const EpiFusionParams *p) {
    if (p->variant == EPI_VARIANT_WARP) return false;
    if (p->variant == EPI_VARIANT_SECTOR && p->sample_locs_in != nullptr) return false;
    return epi::fusion_tile_shape_ok(p->C, p->H, p->W, p->K, p->sample_locs_in != nullptr);
}

// Sizes: `ref_map` is one fp32 copy of the N reference items, `map` one fp32 map of the S·N pairs (source items, fused features).
// The reference planes are staged once however many sources they are fused with.  One bf16 plane of a map is half its fp32 bytes.
// The views form stages its V·N items once (`ref_map`): they are both the query and the source planes, and `map` covers the
// V·S·N pairs' fused features only.
Plan make_plan(const EpiFusionParams *p, const epi::ViewSources &vs, bool head = false) {
    Plan pl;
    const bool views = p->n_views != 0;
    const size_t NP = (size_t)n_pairs(p, vs), px = (size_t)p->H * p->W;
    const size_t ref_map = (size_t)n_ref_items(p) * p->C * px * sizeof(float), map = NP * p->C * px * sizeof(float);
    const size_t src_map_bytes = (size_t)n_src_items(p) * p->C * px * sizeof(float);
    const size_t order_bytes = NP * px * sizeof(uint16_t), geom_bytes = NP * sizeof(epi::PairGeom);
    const bool lowp = map_dtype(p) != EPI_DTYPE_F32, has_z = p->z_weight_folded != nullptr;
    // a 16-bit `out` is rounded by an epilogue pass from an fp32 plane: the fused kernels store fp32 only
    const bool out16 = out_dtype(p) != EPI_DTYPE_F32;
    // sector tiles (pixels grouped by epipolar angle) need the fused geometry; injected locations and an explicit
    // EPI_VARIANT_TILE request use the 4x8 block tiles
    if (want_pipe(p)) pl.kernel = Kernel::Pipe;
    else if (want_tile(p)) pl.kernel = p->variant != EPI_VARIANT_TILE && p->sample_locs_in == nullptr ? Kernel::Sector : Kernel::Tile;
    if (p->variant == EPI_VARIANT_PIPE && pl.kernel != Kernel::Pipe) pl.refusal = "pipe variant does not support this shape";
    if (p->variant == EPI_VARIANT_TILE && pl.kernel != Kernel::Tile) pl.refusal = "tile variant does not support this shape";
    if (p->variant == EPI_VARIANT_SECTOR && pl.kernel != Kernel::Sector)
        pl.refusal = "sector variant does not support this shape / injected locations";

    Regions ws;
    if (pl.kernel == Kernel::Pipe) {
        // without z the fused kernel writes a channels-last, 16-byte-aligned `out` with 16-byte stores; any other `out` gets a
        // pixel-major plane and the transposition pass, which checks the alignment of each store itself
        const bool out_direct = p->out_stride[1] == 1 && p->out_stride[3] % 4 == 0 && p->out_stride[2] % 4 == 0 && p->out_stride[0] % 4 == 0 &&
                                reinterpret_cast<uintptr_t>(p->out) % 16 == 0;
        pl.staging = Staging::Pipe;
        pl.epilogue = head ? Epilogue::Head
                    : has_z ? (epi::zgemm_supported(p->C) ? Epilogue::ZGemm : Epilogue::ZFp32)
                            : (out_direct && !out16 ? Epilogue::Direct : Epilogue::Unstage);
        if (lowp && pl.epilogue == Epilogue::ZFp32 && p->add_ref_residual) pl.ref_copy = RefCopy::After;   // the fp32 z epilogue's residual
        pl.cached = p->cache != nullptr;
        pl.item_px = g_items32 ? 32 : epi::fusion_pipe_item_pixels(p->C, p->H, p->W);
        // [ref_hi | ref_lo | src_hi | src_lo] bf16 planes; bf16 maps have no lo part: [ref_hi | src_hi]
        const bool lo = map_dtype(p) != EPI_DTYPE_BF16;
        pl.ref_hi = ws.part(ref_map / 2);
        if (lo) pl.ref_lo = ws.part(ref_map / 2);
        if (!views) {
            pl.src_hi = ws.part(map / 2);
            if (lo) pl.src_lo = ws.part(map / 2);
        }
        ws.close();
        // fused feature: bf16 (hi, lo) planes for the z GEMM; fp32, contiguous NCHW for the z epilogue, pixel-major for the
        // transposition and the head
        if (pl.epilogue == Epilogue::ZGemm) { pl.fused = ws.part(map / 2); pl.fused_lo = ws.take(map / 2); }
        else if (pl.epilogue != Epilogue::Direct) pl.fused = ws.take(map);
        pl.counter = ws.take(256);
        // folded z weight (+ I with ZRESIDUAL) as bf16 (hi, lo) planes, written by the staging launch
        if (pl.epilogue == Epilogue::ZGemm) { pl.w_hi = ws.part((size_t)p->C * p->C * 2); pl.w_lo = ws.take((size_t)p->C * p->C * 2); }
        if (pl.ref_copy == RefCopy::After) pl.ref32 = ws.take(ref_map);
        Regions cache;
        pl.key = cache.take(NP * 32 * sizeof(float));
        const size_t cache_geom = cache.take(geom_bytes), cache_order = cache.take(order_bytes);
        pl.n_records = epi::fusion_pipe_plan_records((int)NP, p->N, p->H, p->W);       // N: the pairs of one source (or view pair)
        pl.records = cache.take((size_t)pl.n_records * epi::fusion_pipe_plan_record_bytes());
        pl.cache_bytes = cache.end;
        if (pl.cached) { pl.geom = cache_geom; pl.order = cache_order; }
        else { pl.order = ws.take(order_bytes); pl.geom = ws.take(geom_bytes); }      // rebuilt every call
    } else {
        // the tile kernel reads bf16 (hi, lo) planes; the warp kernel reads a channels-last fp32 source in place
        const bool tiles = pl.kernel != Kernel::Warp;
        pl.staging = tiles ? Staging::Planes : (!src_is_channels_last(p) || lowp ? Staging::Nhwc : Staging::InPlace);
        pl.epilogue = head ? Epilogue::Head : has_z ? Epilogue::ZFp32 : out16 ? Epilogue::Unstage : Epilogue::Direct;
        pl.ref_copy = lowp ? RefCopy::Before : RefCopy::None;        // these kernels read the query (and the residual) as fp32
        // views form: a low-precision map's fp32 copy is the warp kernel's source as it stands, and the sector tiles query the
        // source planes
        if (views && lowp && !tiles) pl.staging = Staging::InPlace;
        if (lowp) pl.ref32 = ws.take(ref_map);
        if (tiles) { pl.src_hi = ws.part(src_map_bytes / 2); pl.src_lo = ws.take(src_map_bytes / 2); }
        else if (pl.staging == Staging::Nhwc) pl.src_nhwc = ws.take(src_map_bytes);
        if (pl.epilogue != Epilogue::Direct) pl.fused = ws.take(map);      // NCHW for the z epilogue, pixel-major for the transposition / head
        if (tiles) pl.counter = ws.take(256);
        if (pl.kernel == Kernel::Sector) {
            if (!views) { pl.ref_hi = ws.part(ref_map / 2); pl.ref_lo = ws.take(ref_map / 2); }
            pl.order = ws.take(order_bytes);
        }
    }
    pl.workspace_bytes = ws.end;
    return pl;
}

// a null pointer (an absent optional buffer) or one that (x, y) float pairs can be loaded from and stored to as float2
inline bool aligned8(const void *q) { return reinterpret_cast<uintptr_t>(q) % 8 == 0; }

// the size queries answer 0 for params no plan is made for
bool plannable(const EpiFusionParams *p, const epi::ViewSources &vs) {
    return p && p->N > 0 && p->C > 0 && p->H > 0 && p->W > 0 && p->n_src >= 0 && out_dtype_ok(p) &&
           (p->n_views == 0 || (p->n_views >= 2 && p->n_views <= 256 && p->n_src <= 1 && n_pairs64(p, vs) <= 65535));
}

// Reads the caller's [V][S] host table of V = n_views views into `vs` (the kernels' by-value copy).  Returns null, or why the
// table is refused.
const char *read_table(int V, const int32_t *sources, int32_t S, epi::ViewSources &vs, char *msg, size_t len) {
    if (!sources) return "sources_host is null";
    if (S < 1) return "S (sources per view) must be >= 1";
    if (V < 2) return "the source-table form needs n_views >= 2 (the views of a frame)";
    if ((int64_t)V * S > EPI_VIEW_SOURCES_MAX)
        return "n_views * S must be <= EPI_VIEW_SOURCES_MAX (256): the table travels in the kernels' launch parameters";
    vs.S = S;
    for (int i = 0; i < V * S; i++) {
        const int32_t u = sources[i];
        if (u < 0 || u >= V) { snprintf(msg, len, "sources[%d][%d] = %d is not a view in [0, %d)", i / S, i % S, (int)u, V); return msg; }
        if (u == i / S) { snprintf(msg, len, "sources[%d][%d] = %d pairs view %d with itself", i / S, i % S, (int)u, (int)u); return msg; }
        vs.src[i] = (uint8_t)u;
    }
    return nullptr;
}

const char *read_view_table(const EpiFusionParams *p, const int32_t *sources, int32_t S, epi::ViewSources &vs, char *msg, size_t len) {
    return p ? read_table(p->n_views, sources, S, vs, msg, len) : "params is null";
}

// head: a heat-map call, which has no `out` (epi_fusion_heatmaps_f32 checks that it is null)
int validate(const EpiFusionParams *p, const epi::ViewSources &vs, bool head = false) {
    if (!p) return fail(EPI_EINVAL, "params is null");
    if (p->n_views < 0 || p->n_views == 1) return fail(EPI_EINVAL, "n_views must be 0 or >= 2 (every view against every other)");
    if (p->n_views) {
        if (p->feat_src || p->P_src) return fail(EPI_EINVAL, "n_views >= 2: feat_src and P_src must be null (feat_ref / P_ref hold the views)");
        if (p->n_src > 1) return fail(EPI_EINVAL, "n_views >= 2 needs n_src 0 or 1");
        if (!p->feat_ref || (!p->out && !head)) return fail(EPI_EINVAL, "feat_ref/out must be non-null");
        if (!p->sample_locs_in && !p->P_ref) return fail(EPI_EINVAL, "P_ref required without sample_locs_in");
    } else {
        if (!p->feat_ref || !p->feat_src || (!p->out && !head)) return fail(EPI_EINVAL, "feat_ref/feat_src/out must be non-null");
        if (!p->sample_locs_in && (!p->P_ref || !p->P_src)) return fail(EPI_EINVAL, "P_ref/P_src required without sample_locs_in");
    }
    if (p->N <= 0 || p->C <= 0 || p->H < 2 || p->W < 2) return fail(EPI_EINVAL, "need N,C >= 1 and H,W >= 2");
    if (p->K < 2 || p->K > 256) return fail(EPI_EINVAL, "K (SAMPLESIZE) must be in [2,256]");
    if (p->C > 1024 || (p->C > 512 && p->C % 4 != 0)) return fail(EPI_EINVAL, "C must be <= 512, or <= 1024 and a multiple of 4");
    if (!(p->downsample > 0.f) || !(p->img_scale > 0.f)) return fail(EPI_EINVAL, "downsample and img_scale must be positive");
    if (p->z_weight_folded && !p->z_bias_folded) return fail(EPI_EINVAL, "z_bias_folded required with z_weight_folded");
    if (p->variant < EPI_VARIANT_AUTO || p->variant > EPI_VARIANT_PIPE) return fail(EPI_EINVAL, "unknown variant");
    if (p->feat_dtype & ~0xffff) return fail(EPI_EINVAL, "unknown feat_dtype: bits above 15 must be zero (bits 0-7: the maps' EPI_DTYPE_*, bits 8-15: EPI_OUT_DTYPE of out)");
    if (map_dtype(p) > EPI_DTYPE_F16) return fail(EPI_EINVAL, "unknown feat_dtype");
    if (out_dtype(p) > EPI_DTYPE_F16) return fail(EPI_EINVAL, "unknown output dtype in feat_dtype bits 8-15 (EPI_OUT_DTYPE of EPI_DTYPE_F32, _BF16 or _F16)");
    if (p->n_src < 0) return fail(EPI_EINVAL, "n_src must be >= 0 (0 or 1: one source view per reference item)");
    if (p->n_src > 1 || p->n_views) {
        // the layout, transposition and z epilogue kernels put the item in the grid's z dimension; the pipelined kernel numbers
        // its per-pair work records, and the staging kernel its tiles, in 32-bit ints
        const int64_t np = p->n_views > 256 ? INT64_MAX : n_pairs64(p, vs), hw = (int64_t)p->H * p->W;
        if (np > 65535) return fail(EPI_EINVAL, "pairs (n_src * N, or n_views * S * N with S = n_views - 1 or the table's width) must be <= 65535 (grid z dimension of the per-item kernels)");
        if (np * ((hw + 31) / 32 + 1) + np / p->N * 256 > INT32_MAX || 2 * np * ((hw + 63) / 64) * ((p->C + 63) / 64) > INT32_MAX || np * hw > INT32_MAX)
            return fail(EPI_EINVAL, "pairs * H * W too large: per-pair work records and staging tiles are counted in int32");
    }
    if (p->z_weight_folded && (reinterpret_cast<uintptr_t>(p->z_weight_folded) % 16 != 0 || reinterpret_cast<uintptr_t>(p->z_bias_folded) % 4 != 0))
        return fail(EPI_EINVAL, "z_weight_folded must be 16-byte aligned (contiguous [C,C]) and z_bias_folded 4-byte aligned");
    // every kernel reads and writes the (x, y) pairs of these three as one 8-byte vector
    if (!aligned8(p->sample_locs_in) || !aligned8(p->sample_locs_out) || !aligned8(p->corr_pos))
        return fail(EPI_EINVAL, "sample_locs_in, sample_locs_out and corr_pos must be 8-byte aligned (whole (x, y) float pairs)");
    return EPI_OK;
}

int validate_bwd(const EpiFusionBwdParams *p) {
    if (!p) return fail(EPI_EINVAL, "params is null");
    if (!p->feat_ref || !p->feat_src || !p->attn || !p->grad_out) return fail(EPI_EINVAL, "feat_ref/feat_src/attn/grad_out must be non-null");
    if (!p->sample_locs_in && (!p->P_ref || !p->P_src)) return fail(EPI_EINVAL, "P_ref/P_src required without sample_locs_in");
    if (p->N <= 0 || p->C <= 0 || p->H < 2 || p->W < 2 || p->K < 2 || p->K > 256) return fail(EPI_EINVAL, "bad shape");
    if (p->C > 512 || (p->C > 128 && p->C % 4 != 0)) return fail(EPI_EINVAL, "backward supports C <= 128, or C <= 512 with C % 4 == 0");
    if (p->feat_dtype < EPI_DTYPE_F32 || p->feat_dtype > EPI_DTYPE_F16) return fail(EPI_EINVAL, "unknown feat_dtype");
    if (p->deterministic != 0 && p->deterministic != 1) return fail(EPI_EINVAL, "deterministic must be 0 or 1");
    if (!aligned8(p->sample_locs_in)) return fail(EPI_EINVAL, "sample_locs_in must be 8-byte aligned (whole (x, y) float pairs)");
    return EPI_OK;
}

// Backward workspace: pixel-major copy of feat_src + pixel-major accumulator of its gradient; low-precision maps: + a channels-last
// fp32 copy of feat_ref and a pixel-major fp32 buffer of its gradient (rounded once to the maps' type by the transposition pass);
// deterministic: + the int64 fixed-point accumulator of dL/dfeat_src, one bound word per pair and the [N,K,H·W] float2
// coefficients (accumulator and words adjacent, so that one memset zeroes both)
struct BwdPlan { size_t map, src, dsrc, ref32 = NONE, gref32 = NONE, acc = NONE, words = NONE, coef = NONE, workspace_bytes; };

BwdPlan make_bwd_plan(const EpiFusionBwdParams *p) {
    BwdPlan pl;
    Regions ws;
    pl.map = (size_t)p->N * p->C * p->H * p->W * sizeof(float);
    pl.src = ws.take(pl.map); pl.dsrc = ws.take(pl.map);
    if (p->feat_dtype != EPI_DTYPE_F32) { pl.ref32 = ws.take(pl.map); pl.gref32 = ws.take(pl.map); }
    if (p->deterministic == 1) {
        const size_t px = (size_t)p->N * p->H * p->W;
        pl.acc = ws.take(2 * pl.map);
        pl.words = ws.take((size_t)p->N * sizeof(uint32_t));
        pl.coef = ws.take(px * p->K * sizeof(float2));
    }
    pl.workspace_bytes = ws.end;
    return pl;
}

// Views form of the backward (epi_fusion_views_backward_f32), V·N view items and NP = V·S·N pairs: a pixel-major fp32 copy of
// the view maps (the query and the source map of every pair), the per-item sums (float accumulator of the source terms, then
// dL/dfeats in fp32), one pixel-major fp32 query term per pair; deterministic: + the int64 fixed-point accumulator per item, one
// bound word per item and the [NP,K,H·W] float2 coefficients (accumulator and words adjacent, so that one memset zeroes both)
struct ViewsBwdPlan { size_t items, nhwc, gsum, gq, acc = NONE, words = NONE, coef = NONE, workspace_bytes; };

ViewsBwdPlan make_views_bwd_plan(const EpiFusionBwdParams *p, int V, int S) {
    ViewsBwdPlan pl;
    Regions ws;
    const size_t px = (size_t)p->H * p->W, item = (size_t)p->C * px * sizeof(float), NI = (size_t)V * p->N, NP = NI * S;
    pl.items = NI * item;
    pl.nhwc = ws.take(pl.items); pl.gsum = ws.take(pl.items); pl.gq = ws.take(NP * item);
    if (p->deterministic == 1) {
        pl.acc = ws.take(2 * pl.items);
        pl.words = ws.take(NI * sizeof(uint32_t));
        pl.coef = ws.take(NP * px * p->K * sizeof(float2));
    }
    pl.workspace_bytes = ws.end;
    return pl;
}

// The table (or the all-others form: sources NULL and S = 0) and the params of a views backward.  Returns null, or why they are
// refused; on success `vs` holds the table and `S` the sources per view.
const char *read_views_bwd(const EpiFusionBwdParams *p, int32_t V, const int32_t *sources, int32_t &S, epi::ViewSources &vs,
                           char *msg, size_t len) {
    if (!p) return "params is null";
    if (V < 2) return "n_views must be >= 2 (the views of a frame)";
    if (sources || S != 0) {
        if (const char *why = read_table(V, sources, S, vs, msg, len)) return why;
    } else {
        if (V > 256) return "n_views must be <= 256";
        S = V - 1;
    }
    if (p->N <= 0 || p->H <= 0 || p->W <= 0) return "bad shape";
    const int64_t np = (int64_t)V * S * p->N;
    if (np > 65535) return "pairs (n_views * S * N, S = n_views - 1 or the table's width) must be <= 65535";
    if (np * (((int64_t)p->H * p->W + 31) / 32) > INT32_MAX) return "pairs * H * W too large: the backward's tiles are counted in int32";
    return nullptr;
}

epi::GeomCfg make_geom(int H, int W, int K, float ds, float r, float eps, int correct, int align) {
    epi::GeomCfg g;
    g.ds = ds; g.r = r; g.eps = eps;
    g.xmin = epi::pix2coord(0, ds, r); g.xmax = epi::pix2coord(W - 1, ds, r);
    g.ymin = epi::pix2coord(0, ds, r); g.ymax = epi::pix2coord(H - 1, ds, r);
    g.correct = correct; g.align = align; g.H = H; g.W = W; g.K = K;
    // pix = (v/r + 0.5 - ds/2)/ds ;  g = -1 + 2 pix/(size-1)  |  -1 + 2 (pix+0.5)/size      (multiview.py:25-37,159-163)
    g.inv_rds = (float)(1.0 / ((double)r * ds));
    g.off_ds = (float)((0.5 - (double)ds / 2.0) / ds);
    if (correct) { g.gsx = (float)(2.0 / (W - 1)); g.gox = -1.f; g.gsy = (float)(2.0 / (H - 1)); g.goy = -1.f; }
    else { g.gsx = (float)(2.0 / W); g.gox = (float)(-1.0 + 1.0 / W); g.gsy = (float)(2.0 / H); g.goy = (float)(-1.0 + 1.0 / H); }
    return g;
}

}  // namespace

extern "C" {

int epi_version(void) { return EPI_ABI_VERSION; }

const char *epi_last_error(void) { return g_err; }

int epi_last_launch_count(void) { return g_launches; }

int epi_fusion_backward_deterministic(void) { return 1; }

int epi_fusion_views(void) { return 1; }

int epi_fusion_view_sources(void) { return 1; }

int epi_fusion_views_backward(void) { return 1; }

int epi_kernel_timing_enable(int on) { g_timing = on ? 1 : 0; return EPI_OK; }

// Not declared in the public header: forces the pipe kernel's 32-pixel work items on every shape (on = 1) or restores the
// planned item size (on = 0), so that tests and timings can compare the two on one shape in one process.
int epi_pipe_force_items32(int on) { g_items32 = on ? 1 : 0; return EPI_OK; }

int epi_kernel_timing_last3(float *ms3) {
    if (!ms3) return fail(EPI_EINVAL, "null pointer");
    ms3[0] = ms3[1] = ms3[2] = -1.f;
    if (!g_timing_valid || !g_ev0) return EPI_OK;
    if (cudaEventSynchronize(g_evB) != cudaSuccess) return fail(EPI_ECUDA, "event synchronize failed");
    cudaEventElapsedTime(&ms3[0], g_evA, g_ev0);      // operand staging (+ pixel order)
    cudaEventElapsedTime(&ms3[1], g_ev0, g_ev1);      // fused attention kernel
    cudaEventElapsedTime(&ms3[2], g_ev1, g_evB);      // epilogue pass (z GEMM / output transposition), 0 when there is none
    return EPI_OK;
}

float epi_kernel_timing_last_ms(void) {
    if (!g_timing_valid || !g_ev0) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(g_ev1) != cudaSuccess || cudaEventElapsedTime(&ms, g_ev0, g_ev1) != cudaSuccess) return -1.f;
    return ms;
}

size_t epi_fusion_cache_bytes(const EpiFusionParams *p) { return plannable(p, kAllOthers) ? make_plan(p, kAllOthers).cache_bytes : 0; }

size_t epi_fusion_workspace_bytes(const EpiFusionParams *p) {
    return plannable(p, kAllOthers) ? make_plan(p, kAllOthers).workspace_bytes : 0;
}

}  // extern "C"

namespace {

// h: the head of a heat-map call (epi_fusion_heatmaps_f32, checked there), else null
int forward(const EpiFusionParams *p, const epi::ViewSources &vs, void *stream, const EpiHeadParams *h = nullptr) {
    int rc = validate(p, vs, h != nullptr);
    if (rc != EPI_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const Plan pl = make_plan(p, vs, h != nullptr);
    void *ws = p->workspace;
    if (pl.workspace_bytes > 0 && (!ws || p->workspace_bytes < pl.workspace_bytes)) return fail(EPI_EWORKSPACE, "workspace too small");
    if (pl.workspace_bytes > 0 && reinterpret_cast<uintptr_t>(ws) % 256 != 0) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    g_timing_valid = 0;
    if (g_timing) {
        if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); cudaEventCreate(&g_evA); cudaEventCreate(&g_evB); }
        cudaEventRecord(g_evA, st);
    }
    if (pl.refusal) return fail(EPI_EINVAL, "%s", pl.refusal);
    if (pl.cached) {
        if (p->cache_bytes < pl.cache_bytes) return fail(EPI_EWORKSPACE, "cache too small");
        if (reinterpret_cast<uintptr_t>(p->cache) % 256 != 0) return fail(EPI_EINVAL, "cache must be 256-byte aligned");
    }

    const int dt = map_dtype(p), od = out_dtype(p);
    const int NP = n_pairs(p, vs);      // pairs: items of every output (and of feat_src unless n_views)
    const int NR = n_ref_items(p), V = p->n_views;
    const float *P_src = V ? p->P_ref : p->P_src;      // the views form takes both cameras of a pair from P_ref
    epi::FusionArgs a;
    memset(&a, 0, sizeof(a));
    a.feat_ref = static_cast<const float *>(p->feat_ref); a.ref_dtype = dt;
    a.P_ref = p->P_ref; a.P_src = P_src; a.locs_in = p->sample_locs_in;
    a.attn = p->attn; a.corr_pos = p->corr_pos; a.locs_out = p->sample_locs_out;
    a.N = NP; a.n_ref = p->N; a.n_views = V; a.C = p->C; a.softmax_scale = p->softmax_scale; a.item_px = pl.item_px;
    for (int i = 0; i < 4; i++) a.ref_stride[i] = p->ref_stride[i];
    a.geom = make_geom(p->H, p->W, p->K, p->downsample, p->img_scale, p->eps, p->correct_normalize, p->align_corners);
    float *ref32 = at<float>(ws, pl.ref32);
    const int64_t cl_stride[4] = {(int64_t)p->C * p->H * p->W, 1, (int64_t)p->W * p->C, p->C};      // channels-last / pixel-major
    Launches run;

    // operand staging (first timing group)
    if (pl.ref_copy == RefCopy::Before) {
        if ((rc = run("reference conversion", epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, NR, p->C, p->H, p->W, dt, st)))) return rc;
        a.feat_ref = ref32; a.ref_dtype = EPI_DTYPE_F32;
        for (int i = 0; i < 4; i++) a.ref_stride[i] = cl_stride[i];
    }
    if (pl.staging == Staging::Pipe) {
        const bool have_P = p->P_ref && P_src;
        void *pairs = pl.cached ? p->cache : ws;
        uint16_t *order = have_P ? at<uint16_t>(pairs, pl.order) : nullptr;
        epi::PairGeom *pg = at<epi::PairGeom>(pairs, pl.geom);
        float *okey = pl.cached && have_P ? at<float>(p->cache, pl.key) : nullptr;
        if (okey) {                        // cached work items of the fused kernel, valid per pair for the epoch stored in key slot 31
            a.plan_cache = at<uint8_t>(p->cache, pl.records);
            a.plan_records = pl.n_records;
            a.pair_epoch = reinterpret_cast<const uint32_t *>(okey) + 31;
        }
        int *words = at<int>(ws, pl.counter);
        __nv_bfloat16 *w_hi = at<__nv_bfloat16>(ws, pl.w_hi);
        int kernels = 0;
        const cudaError_t e = epi::launch_stage(p->feat_ref, p->ref_stride, p->feat_src, p->src_stride, dt, at<__nv_bfloat16>(ws, pl.ref_hi),
                                                p->P_ref, P_src, pg, order, okey, w_hi ? p->z_weight_folded : nullptr, w_hi,
                                                p->z_residual ? 1 : 0, words, NP, p->N, V, vs, p->C, p->H, p->W, a.geom, st, kernels);
        if ((rc = run("operand staging", e, kernels))) return rc;
        a.ref_hi = at<__nv_bfloat16>(ws, pl.ref_hi); a.ref_lo = at<__nv_bfloat16>(ws, pl.ref_lo);
        a.src_hi = V ? a.ref_hi : at<__nv_bfloat16>(ws, pl.src_hi); a.src_lo = V ? a.ref_lo : at<__nv_bfloat16>(ws, pl.src_lo);
        a.order = order; a.pair_geom = pg; a.tile_counter = words; a.err_flag = words + 1;
    } else if (pl.staging == Staging::Planes) {
        __nv_bfloat16 *hi = at<__nv_bfloat16>(ws, pl.src_hi), *lo = at<__nv_bfloat16>(ws, pl.src_lo);
        a.tile_counter = at<int>(ws, pl.counter);
        if ((rc = run("operand staging", epi::launch_split_planes(src_map(p), src_strides(p), hi, lo, n_src_items(p), p->C, p->H, p->W, a.tile_counter, dt, st))))
            return rc;
        a.src_hi = hi; a.src_lo = lo;
        if (pl.kernel == Kernel::Sector) {
            // the views form queries the source planes: the split of a bf16 / fp16 value equals that of its fp32 copy
            __nv_bfloat16 *rhi = V ? hi : at<__nv_bfloat16>(ws, pl.ref_hi), *rlo = V ? lo : at<__nv_bfloat16>(ws, pl.ref_lo);
            uint16_t *order = at<uint16_t>(ws, pl.order);
            if (!V && (rc = run("reference staging", epi::launch_split_planes(a.feat_ref, a.ref_stride, rhi, rlo, p->N, p->C, p->H, p->W, nullptr, EPI_DTYPE_F32, st))))
                return rc;
            if ((rc = run("sector ordering", epi::launch_sector_order(p->P_ref, P_src, order, NP, p->N, V, vs, a.geom, st)))) return rc;
            a.ref_hi = rhi; a.ref_lo = rlo; a.order = order;
        }
    } else if (pl.staging == Staging::Nhwc) {
        float *nhwc = at<float>(ws, pl.src_nhwc);
        if ((rc = run("layout staging", epi::launch_nchw_to_nhwc(src_map(p), src_strides(p), nhwc, n_src_items(p), p->C, p->H, p->W, dt, st)))) return rc;
        a.src_nhwc = nhwc;
    } else {
        a.src_nhwc = V ? a.feat_ref : static_cast<const float *>(p->feat_src);     // views form: the map itself or its fp32 copy
    }

    // where the fused kernel writes
    if (pl.epilogue == Epilogue::ZGemm) {
        a.out_hi = at<__nv_bfloat16>(ws, pl.fused); a.out_lo = at<__nv_bfloat16>(ws, pl.fused_lo);
    } else if (pl.epilogue != Epilogue::Direct) {    // pixel-major (full 128-byte lines) for the transposition pass and the head, NCHW for the z epilogue
        const int64_t nchw_stride[4] = {(int64_t)p->C * p->H * p->W, (int64_t)p->H * p->W, p->W, 1};
        a.out = at<float>(ws, pl.fused);
        const bool pm = pl.epilogue == Epilogue::Unstage || pl.epilogue == Epilogue::Head;
        for (int i = 0; i < 4; i++) a.out_stride[i] = pm ? cl_stride[i] : nchw_stride[i];
    } else {
        a.out = p->out;
        for (int i = 0; i < 4; i++) a.out_stride[i] = p->out_stride[i];
        a.add_ref = p->add_ref_residual;
    }

    if (g_timing) cudaEventRecord(g_ev0, st);
    const cudaError_t e = pl.kernel == Kernel::Pipe ? epi::launch_fusion_pipe(a, vs, st)
                        : pl.kernel == Kernel::Warp ? epi::launch_fusion_warp(a, vs, st) : epi::launch_fusion_tile(a, vs, st);
    if ((rc = run("fusion kernel", e))) return rc;
    if (g_timing) cudaEventRecord(g_ev1, st);

    // epilogue (third timing group)
    if (pl.ref_copy == RefCopy::After &&
        (rc = run("reference conversion", epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, NR, p->C, p->H, p->W, dt, st)))) return rc;
    if (pl.epilogue == Epilogue::Unstage) {
        if ((rc = run("output transposition", epi::launch_unstage(a.out, p->add_ref_residual ? p->feat_ref : nullptr, dt, p->ref_stride, p->out,
                                                                  od, p->out_stride, NP, p->N, V, vs, p->C, p->H, p->W, st)))) return rc;
    } else if (pl.epilogue == Epilogue::ZGemm) {
        epi::ZGemmArgs z;
        memset(&z, 0, sizeof(z));
        z.x_hi = a.out_hi; z.x_lo = a.out_lo; z.w_hi = at<__nv_bfloat16>(ws, pl.w_hi); z.w_lo = at<__nv_bfloat16>(ws, pl.w_lo);
        z.Wf = p->z_weight_folded; z.bf = p->z_bias_folded;
        z.ref = p->feat_ref; z.ref_dtype = dt; z.y = p->out;
        for (int i = 0; i < 4; i++) { z.y_stride[i] = p->out_stride[i]; z.ref_stride[i] = p->ref_stride[i]; }
        z.N = NP; z.n_ref = p->N; z.n_views = V; z.C = p->C; z.HW = p->H * p->W; z.W = p->W; z.Npad = p->C;
        z.z_residual = p->z_residual; z.add_ref = p->add_ref_residual;
        if ((rc = run("z GEMM", epi::launch_zgemm(z, vs, od, st)))) return rc;
    } else if (pl.epilogue == Epilogue::ZFp32) {
        epi::ZArgs z;
        memset(&z, 0, sizeof(z));
        z.x = a.out;
        for (int i = 0; i < 4; i++) { z.x_stride[i] = a.out_stride[i]; z.y_stride[i] = p->out_stride[i]; z.ref_stride[i] = ref32 ? cl_stride[i] : p->ref_stride[i]; }
        z.ref = ref32 ? ref32 : static_cast<const float *>(p->feat_ref); z.y = p->out; z.Wf = p->z_weight_folded; z.bf = p->z_bias_folded;
        z.N = NP; z.n_ref = p->N; z.n_views = V; z.vsrc = vs; z.C = p->C; z.HW = p->H * p->W; z.W = p->W;
        z.z_residual = p->z_residual; z.add_ref = p->add_ref_residual;
        if ((rc = run("z epilogue", epi::launch_z_epilogue(z, od, st)))) return rc;
    } else if (pl.epilogue == Epilogue::Head) {
        epi::HeadArgs hd;
        memset(&hd, 0, sizeof(hd));
        hd.x = a.out; hd.A = h->A; hd.B = h->B; hd.b = h->b;
        hd.ref = h->B ? p->feat_ref : nullptr; hd.ref_dtype = dt; hd.heat = h->heat;
        for (int i = 0; i < 4; i++) { hd.ref_stride[i] = p->ref_stride[i]; hd.heat_stride[i] = h->heat_stride[i]; }
        hd.N = NP; hd.C = p->C; hd.HW = p->H * p->W; hd.W = p->W; hd.J = h->J; hd.n_ref = p->N; hd.n_views = V;
        if ((rc = run("head", epi::launch_head(hd, vs, od, st)))) return rc;
    }
    if (g_timing) { cudaEventRecord(g_evB, st); g_timing_valid = 1; }
    g_launches = run.n;
    return EPI_OK;
}

}  // namespace

extern "C" {

int epi_fusion_forward_f32(const EpiFusionParams *p, void *stream) { return forward(p, kAllOthers, stream); }

size_t epi_fusion_view_sources_workspace_bytes(const EpiFusionParams *p, const int32_t *sources_host, int32_t S) {
    epi::ViewSources vs{};
    char msg[128];
    return !read_view_table(p, sources_host, S, vs, msg, sizeof(msg)) && plannable(p, vs) ? make_plan(p, vs).workspace_bytes : 0;
}

size_t epi_fusion_view_sources_cache_bytes(const EpiFusionParams *p, const int32_t *sources_host, int32_t S) {
    epi::ViewSources vs{};
    char msg[128];
    return !read_view_table(p, sources_host, S, vs, msg, sizeof(msg)) && plannable(p, vs) ? make_plan(p, vs).cache_bytes : 0;
}

int epi_fusion_view_sources_forward_f32(const EpiFusionParams *p, const int32_t *sources_host, int32_t S, void *stream) {
    epi::ViewSources vs{};
    char msg[128];
    if (const char *why = read_view_table(p, sources_host, S, vs, msg, sizeof(msg))) return fail(EPI_EINVAL, "%s", why);
    return forward(p, vs, stream);
}

}  // extern "C"

namespace {

// The head of a heat-map call and the fields of p it replaces.  Returns null, or why they are refused.
const char *check_head(const EpiFusionParams *p, const EpiHeadParams *h) {
    if (!p) return "params is null";
    if (!h) return "head params are null";
    if (p->out) return "heat-map call: out must be null (heat receives the result; the fused feature is not stored)";
    if (p->z_weight_folded) return "heat-map call: z_weight_folded must be null (fold z / BN into A and b with epi_fold_head_f32)";
    if (p->add_ref_residual) return "heat-map call: add_ref_residual must be 0 (B = the head weight adds the caller's residual)";
    if (!h->A || !h->b || !h->heat) return "heat-map call: A, b and heat must be non-null";
    if (h->J < 1 || h->J > 64) return "heat-map call: J must be in [1, 64]";
    if (h->reserved[0] || h->reserved[1] || h->reserved[2]) return "heat-map call: reserved words must be zero";
    const uintptr_t es = out_dtype(p) == EPI_DTYPE_F32 ? 4 : 2;
    if (reinterpret_cast<uintptr_t>(h->A) % 4 || reinterpret_cast<uintptr_t>(h->B) % 4 || reinterpret_cast<uintptr_t>(h->b) % 4 ||
        reinterpret_cast<uintptr_t>(h->heat) % es)
        return "heat-map call: A, B and b must be 4-byte aligned and heat aligned to its element size";
    return nullptr;
}

// The table of a heat-map call: the caller's [V][S] table, or none (NULL with S = 0: the pair, n_src and all-others views forms).
const char *read_heat_table(const EpiFusionParams *p, const int32_t *sources, int32_t S, epi::ViewSources &vs, char *msg, size_t len) {
    if (!sources && S == 0) return nullptr;
    return read_view_table(p, sources, S, vs, msg, len);
}

// the size queries plan a heat-map call from the shapes alone: J, not the head's pointers
bool heat_plannable(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources, int32_t S, epi::ViewSources &vs) {
    char msg[128];
    return h && h->J >= 1 && h->J <= 64 && !read_heat_table(p, sources, S, vs, msg, sizeof(msg)) && plannable(p, vs);
}

}  // namespace

extern "C" {

int epi_fusion_heatmaps(void) { return 1; }

size_t epi_fusion_heatmaps_workspace_bytes(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S) {
    epi::ViewSources vs{};
    return heat_plannable(p, h, sources_host, S, vs) ? make_plan(p, vs, true).workspace_bytes : 0;
}

size_t epi_fusion_heatmaps_cache_bytes(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S) {
    epi::ViewSources vs{};
    return heat_plannable(p, h, sources_host, S, vs) ? make_plan(p, vs, true).cache_bytes : 0;
}

int epi_fusion_heatmaps_f32(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S, void *stream) {
    epi::ViewSources vs{};
    char msg[128];
    if (const char *why = check_head(p, h)) return fail(EPI_EINVAL, "%s", why);
    if (const char *why = read_heat_table(p, sources_host, S, vs, msg, sizeof(msg))) return fail(EPI_EINVAL, "%s", why);
    return forward(p, vs, stream, h);
}

int epi_fold_head_f32(const float *Wh, const float *bh, const float *Wf, const float *bf, int32_t z_residual, int32_t J, int32_t C,
                      float *A_out, float *b_out, void *stream) {
    if (!Wh || !A_out || !b_out) return fail(EPI_EINVAL, "Wh, A_out and b_out must be non-null");
    if (J < 1 || C < 1) return fail(EPI_EINVAL, "need J >= 1 and C >= 1");
    cudaError_t e = epi::launch_fold_head(Wh, bh, Wf, bf, z_residual ? 1 : 0, J, C, A_out, b_out, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "head fold launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

size_t epi_fusion_backward_workspace_bytes(const EpiFusionBwdParams *p) {
    if (!p || p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0) return 0;
    return make_bwd_plan(p).workspace_bytes;
}

int epi_fusion_backward_f32(const EpiFusionBwdParams *p, void *stream) {
    int rc = validate_bwd(p);
    if (rc != EPI_OK) return rc;
    if (!p->grad_ref && !p->grad_src) return EPI_OK;
    const BwdPlan pl = make_bwd_plan(p);
    void *ws = p->workspace;
    if (!ws || p->workspace_bytes < pl.workspace_bytes) return fail(EPI_EWORKSPACE, "workspace too small");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int dt = p->feat_dtype;
    const bool lowp = dt != EPI_DTYPE_F32;
    float *nhwc = at<float>(ws, pl.src), *dsrc = at<float>(ws, pl.dsrc), *ref32 = at<float>(ws, pl.ref32), *gref32 = at<float>(ws, pl.gref32);
    const int64_t pm_stride[4] = {(int64_t)p->C * p->H * p->W, 1, (int64_t)p->W * p->C, p->C};      // pixel-major / channels-last
    Launches run;
    if ((rc = run("layout staging", epi::launch_nchw_to_nhwc(p->feat_src, p->src_stride, nhwc, p->N, p->C, p->H, p->W, dt, st)))) return rc;
    if (lowp && (rc = run("reference conversion", epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, p->N, p->C, p->H, p->W, dt, st)))) return rc;
    const bool det = p->deterministic == 1 && p->grad_src;      // dL/dfeat_ref alone is the same launch on both paths
    if (p->grad_src) {
        const cudaError_t e = det ? cudaMemsetAsync(at<char>(ws, pl.acc), 0, pl.words + p->N * sizeof(uint32_t) - pl.acc, st)
                                  : cudaMemsetAsync(dsrc, 0, pl.map, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "memset failed: %s", cudaGetErrorString(e));
    }
    epi::BwdArgs a;
    memset(&a, 0, sizeof(a));
    a.feat_ref = lowp ? ref32 : static_cast<const float *>(p->feat_ref); a.src_nhwc = nhwc; a.P_ref = p->P_ref; a.P_src = p->P_src;
    a.locs_in = p->sample_locs_in; a.attn = p->attn; a.grad_out = p->grad_out; a.grad_attn = p->grad_attn;
    a.grad_ref = !p->grad_ref ? nullptr : (lowp ? gref32 : static_cast<float *>(p->grad_ref));
    a.dsrc_nhwc = p->grad_src ? dsrc : nullptr;
    for (int i = 0; i < 4; i++) {
        a.ref_stride[i] = lowp ? pm_stride[i] : p->ref_stride[i]; a.gout_stride[i] = p->gout_stride[i];
        a.gref_stride[i] = lowp ? pm_stride[i] : p->gref_stride[i];
    }
    a.N = p->N; a.C = p->C; a.softmax_scale = p->softmax_scale; a.grad_keys = p->grad_keys; a.grad_vals = p->grad_vals;
    a.geom = make_geom(p->H, p->W, p->K, p->downsample, p->img_scale, p->eps, p->correct_normalize, p->align_corners);
    if (det) {
        a.dsrc_nhwc = nullptr;
        a.coef = at<float2>(ws, pl.coef); a.pair_max = at<unsigned>(ws, pl.words); a.acc = at<long long>(ws, pl.acc);
        int kernels = 0;
        const cudaError_t e = epi::launch_fusion_bwd_det(a, st, kernels);
        if ((rc = run("deterministic backward kernels", e, kernels))) return rc;
        if ((rc = run("fixed-point conversion", epi::launch_acc_to_f32(a.acc, a.pair_max, dsrc, p->N, p->H * p->W, p->C, st)))) return rc;
    } else if ((rc = run("backward kernel", epi::launch_fusion_bwd(a, st)))) {
        return rc;
    }
    if (p->grad_src &&
        (rc = run("gradient transposition", epi::launch_unstage(dsrc, nullptr, EPI_DTYPE_F32, p->gsrc_stride, p->grad_src, dt, p->gsrc_stride,
                                                                p->N, p->N, 0, kAllOthers, p->C, p->H, p->W, st)))) return rc;
    if (p->grad_ref && lowp &&         // fp32 gradient of a low-precision reference map, rounded once to its type
        (rc = run("gradient transposition", epi::launch_unstage(gref32, nullptr, EPI_DTYPE_F32, p->gref_stride, p->grad_ref, dt, p->gref_stride,
                                                                p->N, p->N, 0, kAllOthers, p->C, p->H, p->W, st)))) return rc;
    g_launches = run.n;
    return EPI_OK;
}

size_t epi_fusion_views_backward_workspace_bytes(const EpiFusionBwdParams *p, int32_t n_views, const int32_t *sources_host, int32_t S) {
    epi::ViewSources vs{};
    char msg[128];
    if (read_views_bwd(p, n_views, sources_host, S, vs, msg, sizeof(msg)) || p->C <= 0) return 0;
    return make_views_bwd_plan(p, n_views, S).workspace_bytes;
}

int epi_fusion_views_backward_f32(const EpiFusionBwdParams *p, int32_t n_views, const int32_t *sources_host, int32_t S, void *stream) {
    epi::ViewSources vs{};
    char msg[128];
    if (const char *why = read_views_bwd(p, n_views, sources_host, S, vs, msg, sizeof(msg))) return fail(EPI_EINVAL, "%s", why);
    if (p->feat_src || p->P_src || p->grad_src)
        return fail(EPI_EINVAL, "views backward: feat_src, P_src and grad_src must be null (feat_ref / P_ref / grad_ref hold the views)");
    // every check of the one-pair backward, with the view maps in both roles
    EpiFusionBwdParams q = *p;
    q.feat_src = p->feat_ref; q.P_src = p->P_ref;
    int rc = validate_bwd(&q);
    if (rc != EPI_OK) return rc;
    if (!p->grad_ref) return EPI_OK;
    const ViewsBwdPlan pl = make_views_bwd_plan(p, n_views, S);
    void *ws = p->workspace;
    if (!ws || p->workspace_bytes < pl.workspace_bytes) return fail(EPI_EWORKSPACE, "workspace too small");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int dt = p->feat_dtype, NI = n_views * p->N, NP = NI * S, HW = p->H * p->W;
    const bool has_src = p->grad_keys || p->grad_vals;
    const bool det = p->deterministic == 1 && has_src;          // the query terms alone are the same launch on both paths
    float *nhwc = at<float>(ws, pl.nhwc), *gsum = at<float>(ws, pl.gsum), *gq = at<float>(ws, pl.gq);
    const int64_t pm_stride[4] = {(int64_t)p->C * HW, 1, (int64_t)p->W * p->C, p->C};      // pixel-major / channels-last
    const epi::BwdViews vw{p->N, n_views, vs};
    Launches run;
    // the view maps staged once: the query of the pairs of a view and the source of the pairs that name it
    if ((rc = run("layout staging", epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, nhwc, NI, p->C, p->H, p->W, dt, st)))) return rc;
    if (has_src) {
        const cudaError_t e = det ? cudaMemsetAsync(at<char>(ws, pl.acc), 0, pl.words + NI * sizeof(uint32_t) - pl.acc, st)
                                  : cudaMemsetAsync(gsum, 0, pl.items, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "memset failed: %s", cudaGetErrorString(e));
    }
    epi::BwdArgs a;
    memset(&a, 0, sizeof(a));
    a.feat_ref = nhwc; a.src_nhwc = nhwc; a.P_ref = p->P_ref; a.P_src = p->P_ref;
    a.locs_in = p->sample_locs_in; a.attn = p->attn; a.grad_out = p->grad_out; a.grad_attn = p->grad_attn;
    a.grad_ref = gq;
    a.dsrc_nhwc = has_src && !det ? gsum : nullptr;
    for (int i = 0; i < 4; i++) { a.ref_stride[i] = pm_stride[i]; a.gout_stride[i] = p->gout_stride[i]; a.gref_stride[i] = pm_stride[i]; }
    a.N = NP; a.C = p->C; a.softmax_scale = p->softmax_scale; a.grad_keys = p->grad_keys; a.grad_vals = p->grad_vals;
    a.geom = make_geom(p->H, p->W, p->K, p->downsample, p->img_scale, p->eps, p->correct_normalize, p->align_corners);
    if (det) { a.coef = at<float2>(ws, pl.coef); a.pair_max = at<unsigned>(ws, pl.words); a.acc = at<long long>(ws, pl.acc); }
    int kernels = 0;
    const cudaError_t e = epi::launch_fusion_bwd_views(a, vw, st, det, kernels);
    if ((rc = run(det ? "deterministic backward kernels" : "backward kernel", e, kernels))) return rc;
    if ((rc = run("gradient sum", epi::launch_views_grad_sum(gq, a.dsrc_nhwc, det ? a.acc : nullptr, det ? a.pair_max : nullptr, gsum,
                                                               vw, HW, p->C, st)))) return rc;
    if ((rc = run("gradient transposition", epi::launch_unstage(gsum, nullptr, EPI_DTYPE_F32, p->gref_stride, p->grad_ref, dt, p->gref_stride,
                                                                NI, NI, 0, kAllOthers, p->C, p->H, p->W, st)))) return rc;
    g_launches = run.n;
    return EPI_OK;
}

int epi_sample_locs_f32(const float *P_ref, const float *P_src, float *sample_locs_out, int32_t N, int32_t H,
                        int32_t W, int32_t K, float downsample, float img_scale, float eps,
                        int32_t correct_normalize, void *stream) {
    if (!P_ref || !P_src || !sample_locs_out) return fail(EPI_EINVAL, "null pointer");
    if (N <= 0 || H < 2 || W < 2 || K < 2) return fail(EPI_EINVAL, "bad shape");
    if (!aligned8(sample_locs_out)) return fail(EPI_EINVAL, "sample_locs_out must be 8-byte aligned (whole (x, y) float pairs)");
    epi::GeomCfg g = make_geom(H, W, K, downsample, img_scale, eps, correct_normalize, 0);
    cudaError_t e = epi::launch_sample_locs(P_ref, P_src, sample_locs_out, N, g, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "sample_locs launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

namespace {

// The arguments both peak finders share.  One warp per (b, j), its index counted in int32; R = (int)(radius + 0.5f) in the kernel,
// whose window loop counts to (2R+1)^2 + 31 in int.
int peaks_args(int64_t BJ, int32_t H, int32_t W, float radius) {
    if (BJ <= 0 || H < 2 || W < 2 || !(radius > 0.f)) return fail(EPI_EINVAL, "bad shape or radius");
    if (!std::isfinite(radius)) return fail(EPI_EINVAL, "radius must be finite");
    if (radius >= (float)(EPI_PEAKS_MAX_R + 1) || (int)(radius + 0.5f) > EPI_PEAKS_MAX_R)
        return fail(EPI_EINVAL, "radius too large: R = int(radius + 0.5) must be at most EPI_PEAKS_MAX_R = %s",
                    std::to_string(EPI_PEAKS_MAX_R).c_str());
    if ((int)(radius + 0.5f) < 1) return fail(EPI_EINVAL, "radius must round to at least 1");
    if (BJ > INT32_MAX / 32) return fail(EPI_EINVAL, "B * J too large (one warp per joint, counted in int32)");
    return EPI_OK;
}

}  // namespace

int epi_find_peaks_f32(const float *heatmaps, float *locs, float *scores, int32_t B, int32_t J, int32_t H, int32_t W,
                       float radius, float downsample, float threshold, int32_t int_div, void *stream) {
    if (!heatmaps || !locs || !scores) return fail(EPI_EINVAL, "null pointer");
    if (B <= 0 || J <= 0) return fail(EPI_EINVAL, "bad shape or radius");
    if (int rc = peaks_args((int64_t)B * J, H, W, radius)) return rc;
    cudaError_t e = epi::launch_peaks(heatmaps, locs, scores, B, J, H, W, radius, downsample, threshold, int_div,
                                      reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "peak kernel launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

int epi_find_peaks_best_f32(const float *heat, float *locs, float *scores, int32_t *src_index, int32_t S, int32_t B, int32_t J,
                            int32_t H, int32_t W, float radius, float downsample, float threshold, int32_t int_div, void *stream) {
    if (!heat || !locs || !scores) return fail(EPI_EINVAL, "null pointer");
    if (S <= 0 || B <= 0 || J <= 0) return fail(EPI_EINVAL, "bad shape or radius");
    if (int rc = peaks_args((int64_t)B * J, H, W, radius)) return rc;
    cudaError_t e = epi::launch_peaks_best(heat, locs, scores, src_index, S, B, J, H, W, radius, downsample, threshold, int_div,
                                           reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "peak kernel launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

namespace {

// torch.linspace(-size/2, size/2, n) in float32, as its CPU kernel computes it: each half one fused multiply-add
void rpsm_linspace(double size, int n, float *g) {
    const float start = (float)(-size / 2), end = (float)(size / 2);
    const float step = (end - start) / (float)(n - 1);
    for (int i = 0; i < n; i++) g[i] = i < n / 2 ? std::fma(step, (float)i, start) : std::fma(-step, (float)(n - 1 - i), end);
}

bool rpsm_size_ok(double v) { return std::isfinite(v) && v > 0.0 && v <= 3.0e38; }

// parents[J] -> the tree (one root, every joint reaching it); false with g_err set otherwise
int rpsm_tree(const int32_t *parents, int J, epi::RpsmTree &t) {
    memset(&t, 0, sizeof(t));
    t.J = J;
    t.E = J - 1;
    t.root = -1;
    for (int j = 0; j < J; j++) {
        const int p = parents[j];
        if (p == -1) {
            if (t.root >= 0) return fail(EPI_EINVAL, "parents has more than one root (-1)");
            t.root = j;
        } else if (p < 0 || p >= J || p == j) {
            return fail(EPI_EINVAL, "parents[j] must be -1 (the root) or another joint's index in [0, J)");
        }
        t.parent[j] = (signed char)p;
    }
    if (t.root < 0) return fail(EPI_EINVAL, "parents has no root (-1)");
    int e = 0;
    for (int j = 0; j < J; j++) {
        int d = 0;
        for (int k = j; parents[k] != -1; k = parents[k])
            if (++d >= J) return fail(EPI_EINVAL, "parents is not a tree (a cycle does not reach the root)");
        t.depth[j] = (signed char)d;
        t.max_depth = d > t.max_depth ? d : t.max_depth;
        t.edge[j] = (signed char)(j == t.root ? -1 : e++);
    }
    int k = 0;
    for (int d = 0; d <= t.max_depth; d++)
        for (int j = 0; j < J; j++)
            if (t.depth[j] == d) t.bfs[k++] = (signed char)j;
    return EPI_OK;
}

size_t rpsm_energy_bytes(const EpiRpsmParams *p) {
    const size_t B = (size_t)p->first_nbins * p->first_nbins * p->first_nbins;
    return align_up((size_t)p->N * p->J * B * sizeof(float));
}

}  // namespace

int epi_rpsm(void) { return 1; }

size_t epi_rpsm_workspace_bytes(const EpiRpsmParams *p) {
    if (!p || p->N < 1 || p->J < 1 || p->J > epi::kRpsmMaxJoints || p->first_nbins < 2 || p->first_nbins > epi::kRpsmMaxNbins0)
        return 0;
    const size_t B = (size_t)p->first_nbins * p->first_nbins * p->first_nbins;
    return rpsm_energy_bytes(p) + align_up((size_t)p->N * (p->J - 1) * B * sizeof(int16_t));
}

int epi_rpsm_f32(const EpiRpsmParams *p, void *stream) {
    if (!p) return fail(EPI_EINVAL, "params must be non-null");
    if (!p->heat || !p->P || !p->crop || !p->root || !p->limb_length || !p->pairwise || !p->parents || !p->pose || !p->workspace)
        return fail(EPI_EINVAL, "heat, P, crop, root, limb_length, pairwise, parents, pose and workspace must be non-null");
    if (p->V < 2 || p->V > 64) return fail(EPI_EINVAL, "V must be in [2, 64]");
    if (p->N < 1) return fail(EPI_EINVAL, "need N >= 1");
    if (p->J < 1 || p->J > epi::kRpsmMaxJoints) return fail(EPI_EINVAL, "J must be in [1, 32]");
    if (p->first_nbins < 2 || p->first_nbins > epi::kRpsmMaxNbins0) return fail(EPI_EINVAL, "first_nbins must be in [2, 16]");
    if (p->recur_nbins < 2 || p->recur_nbins > epi::kRpsmMaxNbinsR) return fail(EPI_EINVAL, "recur_nbins must be in [2, 4]");
    if (p->recur_depth < 0 || p->recur_depth > epi::kRpsmMaxDepth) return fail(EPI_EINVAL, "recur_depth must be in [0, 32]");
    if (p->h < 2 || p->w < 2) return fail(EPI_EINVAL, "the heat-maps need h >= 2 and w >= 2");
    if (!rpsm_size_ok(p->grid_size) || !rpsm_size_ok(p->tolerance))
        return fail(EPI_EINVAL, "grid_size and tolerance must be finite and positive");
    if (!rpsm_size_ok(p->image_size[0]) || !rpsm_size_ok(p->image_size[1]))
        return fail(EPI_EINVAL, "image_size must be finite and positive");
    const void *f32[] = {p->heat, p->P, p->crop, p->root, p->limb_length, p->pairwise, p->pose};
    for (const void *q : f32)
        if (reinterpret_cast<uintptr_t>(q) % 4) return fail(EPI_EINVAL, "heat, P, crop, root, limb_length, pairwise and pose must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(p->workspace) % 256) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    if (p->workspace_bytes < epi_rpsm_workspace_bytes(p)) return fail(EPI_EINVAL, "workspace_bytes is smaller than epi_rpsm_workspace_bytes()");
    epi::RpsmTree t;
    if (int rc = rpsm_tree(p->parents, p->J, t)) return rc;
    epi::RpsmArgs a;
    memset(&a, 0, sizeof(a));
    a.heat = p->heat; a.P = p->P; a.crop = p->crop; a.root = p->root; a.limb = p->limb_length; a.mask = p->pairwise;
    a.energy = static_cast<float *>(p->workspace);
    a.state = at<int16_t>(p->workspace, rpsm_energy_bytes(p));
    a.pose = p->pose;
    a.V = p->V; a.N = p->N; a.h = p->h; a.w = p->w;
    a.n0 = p->first_nbins; a.B = a.n0 * a.n0 * a.n0; a.nr = p->recur_nbins; a.depth = p->recur_depth; a.align = p->align_corners ? 1 : 0;
    a.img0 = p->image_size[0]; a.img1 = p->image_size[1]; a.tol = (float)p->tolerance;
    rpsm_linspace(p->grid_size, a.n0, a.g0);
    double size = p->grid_size / p->first_nbins;          // the reference's cur_grd_size, a Python float
    for (int r = 0; r < a.depth; r++) {
        rpsm_linspace(size, a.nr, a.gr[r]);
        size = size / p->recur_nbins;
    }
    int n = 0;
    cudaError_t e = epi::launch_rpsm(a, t, reinterpret_cast<cudaStream_t>(stream), &n);
    if (e != cudaSuccess) return fail(EPI_ECUDA, "rpsm launch failed: %s", cudaGetErrorString(e));
    g_launches = n;
    return EPI_OK;
}

int epi_rpsm_pairwise_pack(const float *dense, const float *limb_length, int32_t E, int32_t nbins, double grid_size,
                           double tolerance, uint32_t *packed, void *stream) {
    if ((dense == nullptr) == (limb_length == nullptr)) return fail(EPI_EINVAL, "give exactly one of dense and limb_length");
    if (!packed) return fail(EPI_EINVAL, "packed must be non-null");
    if (E < 0 || E > epi::kRpsmMaxJoints - 1) return fail(EPI_EINVAL, "E must be in [0, 31]");
    if (nbins < 2 || nbins > epi::kRpsmMaxNbins0) return fail(EPI_EINVAL, "nbins must be in [2, 16]");
    if (!rpsm_size_ok(grid_size)) return fail(EPI_EINVAL, "grid_size must be finite and positive");
    if (limb_length && !rpsm_size_ok(tolerance)) return fail(EPI_EINVAL, "tolerance must be finite and positive");
    if (reinterpret_cast<uintptr_t>(packed) % 4 || reinterpret_cast<uintptr_t>(dense) % 4 || reinterpret_cast<uintptr_t>(limb_length) % 4)
        return fail(EPI_EINVAL, "dense, limb_length and packed must be 4-byte aligned");
    if (E == 0) return EPI_OK;
    float g0[epi::kRpsmMaxNbins0];
    rpsm_linspace(grid_size, nbins, g0);
    cudaError_t e = epi::launch_rpsm_pack(dense, limb_length, E, nbins, g0, (float)tolerance, packed,
                                          reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "rpsm pairwise pack launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

int epi_triangulate(void) { return 1; }

int epi_triangulate_dlt_f64(const float *locs, const float *scores, const void *P, int32_t P_dtype, double conf_thres, int32_t V,
                            int32_t N, int32_t J, double *X, int32_t *n_used, void *stream) {
    if (!locs || !scores || !P || !X || !n_used) return fail(EPI_EINVAL, "locs, scores, P, X and n_used must be non-null");
    if (V < 2 || V > 64) return fail(EPI_EINVAL, "V must be in [2, 64] (the selected views are a 64-bit mask)");
    if (N < 1 || J < 1) return fail(EPI_EINVAL, "need N >= 1 and J >= 1");
    if ((int64_t)N * J > INT32_MAX) return fail(EPI_EINVAL, "N * J must be <= 2^31 - 1 (one thread per problem, counted in int32)");
    if (P_dtype != EPI_DTYPE_F32 && P_dtype != EPI_DTYPE_F64) return fail(EPI_EINVAL, "P_dtype must be EPI_DTYPE_F32 or EPI_DTYPE_F64");
    if (!std::isfinite(conf_thres)) return fail(EPI_EINVAL, "conf_thres must be finite");
    if (conf_thres > 1000.0) return fail(EPI_EINVAL, "conf_thres must be <= 1000 (the view selection steps down from it by 0.05)");
    const uintptr_t pa = P_dtype == EPI_DTYPE_F64 ? 8 : 4;
    if (reinterpret_cast<uintptr_t>(locs) % 8 || reinterpret_cast<uintptr_t>(X) % 8 || reinterpret_cast<uintptr_t>(P) % pa ||
        reinterpret_cast<uintptr_t>(scores) % 4 || reinterpret_cast<uintptr_t>(n_used) % 4)
        return fail(EPI_EINVAL, "locs, X and a float64 P must be 8-byte aligned, scores, n_used and a float32 P 4-byte aligned");
    cudaError_t e = epi::launch_triangulate(locs, scores, P, P_dtype == EPI_DTYPE_F64, conf_thres, V, N, J, X, n_used,
                                            reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "triangulation launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

int epi_fold_z_bn_f32(const float *z_weight, const float *z_bias, const float *bn_weight, const float *bn_bias,
                      const float *bn_mean, const float *bn_var, float bn_eps, int32_t C, float *w_folded,
                      float *b_folded, void *stream) {
    if (!z_weight || !bn_weight || !bn_bias || !bn_mean || !bn_var || !w_folded || !b_folded || C <= 0)
        return fail(EPI_EINVAL, "null pointer or bad C");
    cudaError_t e = epi::launch_fold_z_bn(z_weight, z_bias, bn_weight, bn_bias, bn_mean, bn_var, bn_eps, C, w_folded,
                                          b_folded, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "fold launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

}  // extern "C"
