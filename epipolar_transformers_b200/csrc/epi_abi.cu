// epi_abi.cu — the extern "C" boundary declared in include/epipolar_b200.h.
// Validates arguments, carves the caller's workspace, launches kernels on the caller's stream.
#include <cstdio>
#include <cstring>

#include "../../include/epipolar_b200.h"
#include "epi_kernels.cuh"

namespace {

thread_local char g_err[512] = "";
thread_local int g_launches = 0;
thread_local int g_timing = 0, g_timing_valid = 0;
thread_local cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr, g_evA = nullptr, g_evB = nullptr;   // A: call start, B: call end

int fail(int code, const char *fmt, const char *detail = "") {
    snprintf(g_err, sizeof(g_err), fmt, detail);
    return code;
}

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// source views per reference item (EpiFusionParams.n_src: 0 and 1 both mean one)
inline int n_sources(const EpiFusionParams *p) { return p->n_src > 1 ? p->n_src : 1; }
// (reference, source) pairs = items of feat_src, out, attn, corr_pos and the sample locations
inline int n_pairs(const EpiFusionParams *p) { return n_sources(p) * p->N; }

bool src_is_channels_last(const EpiFusionParams *p) {
    const int64_t *s = p->src_stride;
    const int64_t C = p->C, H = p->H, W = p->W;
    return s[1] == 1 && s[3] == C && s[2] == W * C && (n_pairs(p) == 1 || s[0] == H * W * C) &&
           (reinterpret_cast<uintptr_t>(p->feat_src) % 16 == 0);
}

struct Plan {
    size_t off_src = 0, off_prez = 0, off_counter = 0, off_ref = 0, off_order = 0, off_wplanes = 0, off_geom = 0, off_ref32 = 0, total = 0;
    bool stage_src = false, has_z = false, tile = false, sector = false, pipe = false, unstage = false;
    bool ref32 = false;     // fp32 channels-last copy of a low-precision feat_ref for the kernels that read feat_ref as fp32
};

bool want_pipe(const EpiFusionParams *p) {
    if (p->variant != EPI_VARIANT_AUTO && p->variant != EPI_VARIANT_PIPE) return false;
    if (!epi::fusion_pipe_shape_ok(p->C, p->H, p->W, p->K, p->sample_locs_in != nullptr)) return false;
    // Automatic selection leaves one corner to the other kernels: K > 48 on maps of 2K pixels or more a side.  There a single pixel's
    // taps (4K, sampled sparsely along a long line) already fill the 256-row union, so every work item splits down to one pixel and
    // the per-pixel CUDA-core kernel does less work (tools/gpu_mapsize.py times the kernels per map size).
    if (p->variant == EPI_VARIANT_AUTO && 4 * p->K > 192 && (p->H > p->W ? p->H : p->W) >= 2 * p->K) return false;
    return true;
}

bool want_tile(const EpiFusionParams *p) {
    if (p->variant == EPI_VARIANT_WARP) return false;
    if (p->variant == EPI_VARIANT_SECTOR && p->sample_locs_in != nullptr) return false;
    return epi::fusion_tile_shape_ok(p->C, p->H, p->W, p->K, p->sample_locs_in != nullptr);
}

// Sizes: `ref_map` is one fp32 copy of the N reference items, `map` one fp32 map of the S·N pairs (source items, fused features).
// The reference planes are staged once however many sources they are fused with.
Plan make_plan(const EpiFusionParams *p) {
    Plan pl;
    const size_t ref_map = (size_t)p->N * p->C * p->H * p->W * sizeof(float);
    const size_t map = (size_t)n_pairs(p) * p->C * p->H * p->W * sizeof(float);
    const size_t NP = (size_t)n_pairs(p);
    const bool lowp = p->feat_dtype != EPI_DTYPE_F32;
    pl.pipe = want_pipe(p);
    if (pl.pipe) {
        // [ref_hi | ref_lo | src_hi | src_lo] bf16 planes (bytes of one fp32 reference map + one fp32 source map; bf16 maps:
        // [ref_hi | src_hi], half of that), pre-z planes, pixel order, pair constants
        pl.has_z = p->z_weight_folded != nullptr;
        size_t off = 0;
        pl.off_ref = off; off += align_up(p->feat_dtype == EPI_DTYPE_BF16 ? (ref_map + map) / 2 : ref_map + map);
        // pre-z planes (z path) or the pixel-major fp32 plane the fused kernel writes when the caller's tensor is NCHW
        pl.unstage = !pl.has_z && !(p->out_stride[1] == 1 && p->out_stride[3] % 4 == 0 && p->out_stride[2] % 4 == 0 && p->out_stride[0] % 4 == 0);
        if (pl.has_z || pl.unstage) { pl.off_prez = off; off += align_up(map); }
        pl.off_counter = off; off += 256;
        if (pl.has_z && epi::zgemm_supported(p->C)) { pl.off_wplanes = off; off += align_up((size_t)p->C * p->C * 4); }
        pl.ref32 = lowp && pl.has_z && !epi::zgemm_supported(p->C) && p->add_ref_residual;      // the fp32 z epilogue's residual
        if (pl.ref32) { pl.off_ref32 = off; off += align_up(ref_map); }
        if (!p->cache) {               // no persistent cache: pixel order and pair constants are rebuilt in the workspace every call
            pl.off_order = off; off += align_up(NP * p->H * p->W * sizeof(uint16_t));
            pl.off_geom = off; off += align_up(NP * sizeof(epi::PairGeom));
        }
        pl.total = off;
        return pl;
    }
    pl.tile = want_tile(p);
    // sector tiles (pixels grouped by epipolar angle) need the fused geometry; injected locations and an explicit
    // EPI_VARIANT_TILE request use the 4x8 block tiles
    pl.sector = pl.tile && p->variant != EPI_VARIANT_TILE && p->sample_locs_in == nullptr;
    // tile kernel: bf16 (hi, lo) planes, same bytes as one fp32 map; the warp kernel reads a channels-last fp32 source in place
    pl.stage_src = pl.tile || !src_is_channels_last(p) || lowp;
    pl.has_z = p->z_weight_folded != nullptr;
    pl.ref32 = lowp;                                         // these kernels read the query (and the residual) as fp32
    size_t off = 0;
    if (pl.ref32) { pl.off_ref32 = off; off += align_up(ref_map); }
    if (pl.stage_src) { pl.off_src = off; off += align_up(map); }
    if (pl.has_z) { pl.off_prez = off; off += align_up(map); }
    if (pl.tile) { pl.off_counter = off; off += 256; }
    if (pl.sector) {
        pl.off_ref = off; off += align_up(ref_map);
        pl.off_order = off; off += align_up(NP * p->H * p->W * sizeof(uint16_t));
    }
    pl.total = off;
    return pl;
}

int validate(const EpiFusionParams *p) {
    if (!p) return fail(EPI_EINVAL, "params is null");
    if (!p->feat_ref || !p->feat_src || !p->out) return fail(EPI_EINVAL, "feat_ref/feat_src/out must be non-null");
    if (!p->sample_locs_in && (!p->P_ref || !p->P_src)) return fail(EPI_EINVAL, "P_ref/P_src required without sample_locs_in");
    if (p->N <= 0 || p->C <= 0 || p->H < 2 || p->W < 2) return fail(EPI_EINVAL, "need N,C >= 1 and H,W >= 2");
    if (p->K < 2 || p->K > 256) return fail(EPI_EINVAL, "K (SAMPLESIZE) must be in [2,256]");
    if (p->C > 1024 || (p->C > 512 && p->C % 4 != 0)) return fail(EPI_EINVAL, "C must be <= 512, or <= 1024 and a multiple of 4");
    if (!(p->downsample > 0.f) || !(p->img_scale > 0.f)) return fail(EPI_EINVAL, "downsample and img_scale must be positive");
    if (p->z_weight_folded && !p->z_bias_folded) return fail(EPI_EINVAL, "z_bias_folded required with z_weight_folded");
    if (p->variant < EPI_VARIANT_AUTO || p->variant > EPI_VARIANT_PIPE) return fail(EPI_EINVAL, "unknown variant");
    if (p->feat_dtype < EPI_DTYPE_F32 || p->feat_dtype > EPI_DTYPE_F16) return fail(EPI_EINVAL, "unknown feat_dtype");
    if (p->n_src < 0) return fail(EPI_EINVAL, "n_src must be >= 0 (0 or 1: one source view per reference item)");
    if (p->n_src > 1) {
        // the layout, transposition and z epilogue kernels put the item in the grid's z dimension; the pipelined kernel numbers
        // its per-pair work records, and the staging kernel its tiles, in 32-bit ints
        const int64_t np = (int64_t)p->n_src * p->N, hw = (int64_t)p->H * p->W;
        if (np > 65535) return fail(EPI_EINVAL, "n_src * N must be <= 65535 (grid z dimension of the per-item kernels)");
        if (np * ((hw + 31) / 32 + 1) + p->n_src * 256 > INT32_MAX || 2 * np * ((hw + 63) / 64) * ((p->C + 63) / 64) > INT32_MAX || np * hw > INT32_MAX)
            return fail(EPI_EINVAL, "n_src * N * H * W too large: per-pair work records and staging tiles are counted in int32");
    }
    if (p->z_weight_folded && (reinterpret_cast<uintptr_t>(p->z_weight_folded) % 16 != 0 || reinterpret_cast<uintptr_t>(p->z_bias_folded) % 4 != 0))
        return fail(EPI_EINVAL, "z_weight_folded must be 16-byte aligned (contiguous [C,C]) and z_bias_folded 4-byte aligned");
    return EPI_OK;
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

int epi_kernel_timing_enable(int on) { g_timing = on ? 1 : 0; return EPI_OK; }

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

// per pair: key (32 words), constants, pixel order, work records of the pipelined kernel
size_t epi_fusion_cache_bytes(const EpiFusionParams *p) {
    if (!p || p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0 || p->n_src < 0 || !want_pipe(p)) return 0;
    const size_t NP = (size_t)n_pairs(p);
    return align_up(NP * 32 * sizeof(float)) + align_up(NP * sizeof(epi::PairGeom)) +
           align_up(NP * p->H * p->W * sizeof(uint16_t)) +
           align_up((size_t)epi::fusion_pipe_plan_records((int)NP, p->N, p->H, p->W) * epi::fusion_pipe_plan_record_bytes());
}

size_t epi_fusion_workspace_bytes(const EpiFusionParams *p) {
    if (!p || p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0 || p->n_src < 0) return 0;
    return make_plan(p).total;
}

int epi_fusion_forward_f32(const EpiFusionParams *p, void *stream) {
    int rc = validate(p);
    if (rc != EPI_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const Plan pl = make_plan(p);
    if (pl.total > 0 && (!p->workspace || p->workspace_bytes < pl.total)) return fail(EPI_EWORKSPACE, "workspace too small");
    if (pl.total > 0 && reinterpret_cast<uintptr_t>(p->workspace) % 256 != 0) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    char *ws = static_cast<char *>(p->workspace);
    int launches = 0;
    cudaError_t e;
    const __nv_bfloat16 *w_hi = nullptr, *w_lo = nullptr;
    g_timing_valid = 0;
    if (g_timing) {
        if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); cudaEventCreate(&g_evA); cudaEventCreate(&g_evB); }
        cudaEventRecord(g_evA, st);
    }

    const int dt = p->feat_dtype;
    const int NP = n_pairs(p);          // pairs: items of feat_src and of every output; feat_ref has p->N items
    epi::FusionArgs a;
    memset(&a, 0, sizeof(a));
    a.feat_ref = static_cast<const float *>(p->feat_ref); a.ref_dtype = dt;
    a.P_ref = p->P_ref; a.P_src = p->P_src; a.locs_in = p->sample_locs_in;
    a.attn = p->attn; a.corr_pos = p->corr_pos; a.locs_out = p->sample_locs_out;
    a.N = NP; a.n_ref = p->N; a.C = p->C; a.softmax_scale = p->softmax_scale;
    for (int i = 0; i < 4; i++) a.ref_stride[i] = p->ref_stride[i];
    a.geom = make_geom(p->H, p->W, p->K, p->downsample, p->img_scale, p->eps, p->correct_normalize, p->align_corners);
    // fp32 kernels that read feat_ref get a channels-last fp32 copy of a low-precision map
    float *ref32 = pl.ref32 ? reinterpret_cast<float *>(ws + pl.off_ref32) : nullptr;
    const int64_t ref32_stride[4] = {(int64_t)p->C * p->H * p->W, 1, (int64_t)p->W * p->C, p->C};

    if (p->variant == EPI_VARIANT_PIPE && !pl.pipe) return fail(EPI_EINVAL, "pipe variant does not support this shape");
    if (pl.pipe) {
        const size_t ref_elems = (size_t)p->N * p->C * p->H * p->W, elems = (size_t)NP * p->C * p->H * p->W;
        __nv_bfloat16 *planes = reinterpret_cast<__nv_bfloat16 *>(ws + pl.off_ref);
        int *words = reinterpret_cast<int *>(ws + pl.off_counter);
        const bool have_P = p->P_ref && p->P_src;
        uint16_t *order = nullptr;
        epi::PairGeom *pg = nullptr;
        float *okey = nullptr;
        if (p->cache) {
            if (p->cache_bytes < epi_fusion_cache_bytes(p)) return fail(EPI_EWORKSPACE, "cache too small");
            if (reinterpret_cast<uintptr_t>(p->cache) % 256 != 0) return fail(EPI_EINVAL, "cache must be 256-byte aligned");
            char *cb = static_cast<char *>(p->cache);
            okey = reinterpret_cast<float *>(cb);
            pg = reinterpret_cast<epi::PairGeom *>(cb + align_up((size_t)NP * 32 * sizeof(float)));
            order = reinterpret_cast<uint16_t *>(cb + align_up((size_t)NP * 32 * sizeof(float)) + align_up((size_t)NP * sizeof(epi::PairGeom)));
            if (have_P) {                      // cached work items of the fused kernel, valid per pair for the epoch stored in key slot 31
                a.plan_cache = reinterpret_cast<uint8_t *>(order) + align_up((size_t)NP * p->H * p->W * sizeof(uint16_t));
                a.plan_records = epi::fusion_pipe_plan_records(NP, p->N, p->H, p->W);
                a.pair_epoch = reinterpret_cast<const uint32_t *>(okey) + 31;
            }
        } else {
            order = reinterpret_cast<uint16_t *>(ws + pl.off_order);
            pg = reinterpret_cast<epi::PairGeom *>(ws + pl.off_geom);
        }
        if (!have_P) { order = nullptr; okey = nullptr; }
        const bool z_planes = pl.has_z && epi::zgemm_supported(p->C);
        __nv_bfloat16 *wpl = z_planes ? reinterpret_cast<__nv_bfloat16 *>(ws + pl.off_wplanes) : nullptr;
        e = epi::launch_stage(p->feat_ref, p->ref_stride, p->feat_src, p->src_stride, dt, planes, p->P_ref, p->P_src, pg, order, okey,
                              z_planes ? p->z_weight_folded : nullptr, wpl, p->z_residual ? 1 : 0, words, NP, p->N, p->C, p->H, p->W, a.geom, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "operand staging launch failed: %s", cudaGetErrorString(e));
        launches += (order && (size_t)p->H * p->W * 2 + 16384 > 64 * 1024) ? 2 : 1;      // large maps order their pixels in a launch of their own
        w_hi = wpl; w_lo = wpl ? wpl + (size_t)p->C * p->C : nullptr;
        if (dt == EPI_DTYPE_BF16) { a.ref_hi = planes; a.src_hi = planes + ref_elems; }       // no lo planes: the pipe kernel's LO = false form
        else { a.ref_hi = planes; a.ref_lo = planes + ref_elems; a.src_hi = planes + 2 * ref_elems; a.src_lo = planes + 2 * ref_elems + elems; }
        a.order = order; a.pair_geom = pg; a.tile_counter = words; a.err_flag = words + 1;
    } else
    if (p->variant == EPI_VARIANT_TILE && !pl.tile) return fail(EPI_EINVAL, "tile variant does not support this shape");
    if (p->variant == EPI_VARIANT_SECTOR && !pl.sector) return fail(EPI_EINVAL, "sector variant does not support this shape / injected locations");
    if (!pl.pipe && ref32) {
        e = epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, p->N, p->C, p->H, p->W, dt, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "reference conversion launch failed: %s", cudaGetErrorString(e));
        launches++;
        a.feat_ref = ref32; a.ref_dtype = EPI_DTYPE_F32;
        for (int i = 0; i < 4; i++) a.ref_stride[i] = ref32_stride[i];
    }
    if (pl.tile) {
        __nv_bfloat16 *hi = reinterpret_cast<__nv_bfloat16 *>(ws + pl.off_src);
        __nv_bfloat16 *lo = hi + (size_t)NP * p->C * p->H * p->W;
        a.tile_counter = reinterpret_cast<int *>(ws + pl.off_counter);
        e = epi::launch_split_planes(p->feat_src, p->src_stride, hi, lo, NP, p->C, p->H, p->W, a.tile_counter, dt, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "operand staging launch failed: %s", cudaGetErrorString(e));
        launches++;
        a.src_hi = hi; a.src_lo = lo;
        if (pl.sector) {
            __nv_bfloat16 *rhi = reinterpret_cast<__nv_bfloat16 *>(ws + pl.off_ref);
            __nv_bfloat16 *rlo = rhi + (size_t)p->N * p->C * p->H * p->W;
            e = epi::launch_split_planes(a.feat_ref, a.ref_stride, rhi, rlo, p->N, p->C, p->H, p->W, nullptr, EPI_DTYPE_F32, st);
            if (e != cudaSuccess) return fail(EPI_ECUDA, "reference staging launch failed: %s", cudaGetErrorString(e));
            uint16_t *order = reinterpret_cast<uint16_t *>(ws + pl.off_order);
            e = epi::launch_sector_order(p->P_ref, p->P_src, order, NP, p->N, a.geom, st);
            if (e != cudaSuccess) return fail(EPI_ECUDA, "sector ordering launch failed: %s", cudaGetErrorString(e));
            launches += 2;
            a.ref_hi = rhi; a.ref_lo = rlo; a.order = order;
        }
    } else if (pl.stage_src) {
        float *nhwc = reinterpret_cast<float *>(ws + pl.off_src);
        e = epi::launch_nchw_to_nhwc(p->feat_src, p->src_stride, nhwc, NP, p->C, p->H, p->W, dt, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "layout staging launch failed: %s", cudaGetErrorString(e));
        launches++;
        a.src_nhwc = nhwc;
    } else {
        a.src_nhwc = static_cast<const float *>(p->feat_src);
    }

    const bool z_tc = pl.has_z && pl.pipe && epi::zgemm_supported(p->C);      // tensor-core z GEMM (operand planes come from the staging launch)
    if (z_tc) {         // fused feature leaves the tile kernel as bf16 (hi, lo) planes: the A operand of the z GEMM
        a.out = nullptr;
        a.out_hi = reinterpret_cast<__nv_bfloat16 *>(ws + pl.off_prez);
        a.out_lo = a.out_hi + (size_t)NP * p->C * p->H * p->W;
        a.add_ref = 0;
    } else if (pl.pipe && pl.unstage) {   // fused feature leaves the kernel pixel-major (full 128-byte lines); a transposition pass writes `out`
        a.out = reinterpret_cast<float *>(ws + pl.off_prez);
        a.out_stride[0] = (int64_t)p->C * p->H * p->W; a.out_stride[1] = 1;
        a.out_stride[2] = (int64_t)p->W * p->C; a.out_stride[3] = p->C;
        a.add_ref = 0;
    } else if (pl.has_z) {     // fused feature goes to the pre-z buffer (contiguous NCHW), epilogue writes `out`
        a.out = reinterpret_cast<float *>(ws + pl.off_prez);
        a.out_stride[0] = (int64_t)p->C * p->H * p->W; a.out_stride[1] = (int64_t)p->H * p->W;
        a.out_stride[2] = p->W; a.out_stride[3] = 1;
        a.add_ref = 0;
    } else {
        a.out = p->out;
        for (int i = 0; i < 4; i++) a.out_stride[i] = p->out_stride[i];
        a.add_ref = p->add_ref_residual;
    }

    const bool use_tile = pl.tile && epi::fusion_tile_supported(a);
    if (pl.tile && !use_tile) return fail(EPI_EINVAL, "internal: tile plan without tile support");
    if (g_timing) cudaEventRecord(g_ev0, st);
    e = pl.pipe ? epi::launch_fusion_pipe(a, st) : (use_tile ? epi::launch_fusion_tile(a, st) : epi::launch_fusion_warp(a, st));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "fusion kernel launch failed: %s", cudaGetErrorString(e));
    if (g_timing) cudaEventRecord(g_ev1, st);
    launches++;

    if (pl.pipe && pl.unstage) {
        e = epi::launch_unstage(a.out, p->add_ref_residual ? p->feat_ref : nullptr, dt, p->ref_stride, p->out, EPI_DTYPE_F32, p->out_stride,
                                NP, p->N, p->C, p->H, p->W, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "output transposition launch failed: %s", cudaGetErrorString(e));
        launches++;
    }
    if (z_tc) {
        epi::ZGemmArgs z;
        memset(&z, 0, sizeof(z));
        z.x_hi = a.out_hi; z.x_lo = a.out_lo; z.w_hi = w_hi; z.w_lo = w_lo; z.Wf = p->z_weight_folded; z.bf = p->z_bias_folded;
        z.ref = p->feat_ref; z.ref_dtype = dt; z.y = p->out;
        for (int i = 0; i < 4; i++) { z.y_stride[i] = p->out_stride[i]; z.ref_stride[i] = p->ref_stride[i]; }
        z.N = NP; z.n_ref = p->N; z.C = p->C; z.HW = p->H * p->W; z.W = p->W; z.Npad = p->C;
        z.z_residual = p->z_residual; z.add_ref = p->add_ref_residual;
        e = epi::launch_zgemm(z, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "z GEMM launch failed: %s", cudaGetErrorString(e));
        launches++;
    } else if (pl.has_z) {
        if (pl.pipe && ref32) {            // (the other kernels' plans made the copy before the fused kernel)
            e = epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, p->N, p->C, p->H, p->W, dt, st);
            if (e != cudaSuccess) return fail(EPI_ECUDA, "reference conversion launch failed: %s", cudaGetErrorString(e));
            launches++;
        }
        epi::ZArgs z;
        memset(&z, 0, sizeof(z));
        z.x = a.out;
        for (int i = 0; i < 4; i++) { z.x_stride[i] = a.out_stride[i]; z.y_stride[i] = p->out_stride[i]; z.ref_stride[i] = ref32 ? ref32_stride[i] : p->ref_stride[i]; }
        z.ref = ref32 ? ref32 : static_cast<const float *>(p->feat_ref); z.y = p->out; z.Wf = p->z_weight_folded; z.bf = p->z_bias_folded;
        z.N = NP; z.n_ref = p->N; z.C = p->C; z.HW = p->H * p->W; z.W = p->W;
        z.z_residual = p->z_residual; z.add_ref = p->add_ref_residual;
        e = epi::launch_z_epilogue(z, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "z epilogue launch failed: %s", cudaGetErrorString(e));
        launches++;
    }
    if (g_timing) { cudaEventRecord(g_evB, st); g_timing_valid = 1; }
    g_launches = launches;
    return EPI_OK;
}

size_t epi_fusion_backward_workspace_bytes(const EpiFusionBwdParams *p) {
    if (!p || p->N <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0) return 0;
    const size_t map = (size_t)p->N * p->C * p->H * p->W * sizeof(float);
    // pixel-major copy of feat_src + pixel-major accumulator of its gradient; low-precision maps: + a channels-last fp32 copy of
    // feat_ref and a pixel-major fp32 buffer of its gradient (rounded once to the maps' type by the transposition pass)
    return (p->feat_dtype != EPI_DTYPE_F32 ? 4 : 2) * align_up(map);
}

int epi_fusion_backward_f32(const EpiFusionBwdParams *p, void *stream) {
    if (!p) return fail(EPI_EINVAL, "params is null");
    if (!p->feat_ref || !p->feat_src || !p->attn || !p->grad_out) return fail(EPI_EINVAL, "feat_ref/feat_src/attn/grad_out must be non-null");
    if (!p->sample_locs_in && (!p->P_ref || !p->P_src)) return fail(EPI_EINVAL, "P_ref/P_src required without sample_locs_in");
    if (p->N <= 0 || p->C <= 0 || p->H < 2 || p->W < 2 || p->K < 2 || p->K > 256) return fail(EPI_EINVAL, "bad shape");
    if (p->C > 512 || (p->C > 128 && p->C % 4 != 0)) return fail(EPI_EINVAL, "backward supports C <= 128, or C <= 512 with C % 4 == 0");
    if (p->feat_dtype < EPI_DTYPE_F32 || p->feat_dtype > EPI_DTYPE_F16) return fail(EPI_EINVAL, "unknown feat_dtype");
    if (!p->grad_ref && !p->grad_src) return EPI_OK;
    const size_t need = epi_fusion_backward_workspace_bytes(p);
    if (!p->workspace || p->workspace_bytes < need) return fail(EPI_EWORKSPACE, "workspace too small");
    if (reinterpret_cast<uintptr_t>(p->workspace) % 256 != 0) return fail(EPI_EINVAL, "workspace must be 256-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t map = (size_t)p->N * p->C * p->H * p->W * sizeof(float);
    const int dt = p->feat_dtype;
    const bool lowp = dt != EPI_DTYPE_F32;
    float *nhwc = reinterpret_cast<float *>(p->workspace);
    float *dsrc = reinterpret_cast<float *>(static_cast<char *>(p->workspace) + align_up(map));
    float *ref32 = lowp ? reinterpret_cast<float *>(static_cast<char *>(p->workspace) + 2 * align_up(map)) : nullptr;
    float *gref32 = lowp ? reinterpret_cast<float *>(static_cast<char *>(p->workspace) + 3 * align_up(map)) : nullptr;
    const int64_t pm_stride[4] = {(int64_t)p->C * p->H * p->W, 1, (int64_t)p->W * p->C, p->C};      // pixel-major / channels-last
    cudaError_t e = epi::launch_nchw_to_nhwc(p->feat_src, p->src_stride, nhwc, p->N, p->C, p->H, p->W, dt, st);
    if (e != cudaSuccess) return fail(EPI_ECUDA, "layout staging launch failed: %s", cudaGetErrorString(e));
    int launches = 1;
    if (lowp) {
        e = epi::launch_nchw_to_nhwc(p->feat_ref, p->ref_stride, ref32, p->N, p->C, p->H, p->W, dt, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "reference conversion launch failed: %s", cudaGetErrorString(e));
        launches++;
    }
    if (p->grad_src) {
        e = cudaMemsetAsync(dsrc, 0, map, st);
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
    e = epi::launch_fusion_bwd(a, st);
    if (e != cudaSuccess) return fail(EPI_ECUDA, "backward kernel launch failed: %s", cudaGetErrorString(e));
    launches++;
    if (p->grad_src) {
        e = epi::launch_unstage(dsrc, nullptr, EPI_DTYPE_F32, p->gsrc_stride, p->grad_src, dt, p->gsrc_stride, p->N, p->N, p->C, p->H, p->W, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "gradient transposition launch failed: %s", cudaGetErrorString(e));
        launches++;
    }
    if (p->grad_ref && lowp) {         // fp32 gradient of a low-precision reference map, rounded once to its type
        e = epi::launch_unstage(gref32, nullptr, EPI_DTYPE_F32, p->gref_stride, p->grad_ref, dt, p->gref_stride, p->N, p->N, p->C, p->H, p->W, st);
        if (e != cudaSuccess) return fail(EPI_ECUDA, "gradient transposition launch failed: %s", cudaGetErrorString(e));
        launches++;
    }
    g_launches = launches;
    return EPI_OK;
}

int epi_sample_locs_f32(const float *P_ref, const float *P_src, float *sample_locs_out, int32_t N, int32_t H,
                        int32_t W, int32_t K, float downsample, float img_scale, float eps,
                        int32_t correct_normalize, void *stream) {
    if (!P_ref || !P_src || !sample_locs_out) return fail(EPI_EINVAL, "null pointer");
    if (N <= 0 || H < 2 || W < 2 || K < 2) return fail(EPI_EINVAL, "bad shape");
    epi::GeomCfg g = make_geom(H, W, K, downsample, img_scale, eps, correct_normalize, 0);
    cudaError_t e = epi::launch_sample_locs(P_ref, P_src, sample_locs_out, N, g, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "sample_locs launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

int epi_find_peaks_f32(const float *heatmaps, float *locs, float *scores, int32_t B, int32_t J, int32_t H, int32_t W,
                       float radius, float downsample, float threshold, int32_t int_div, void *stream) {
    if (!heatmaps || !locs || !scores) return fail(EPI_EINVAL, "null pointer");
    if (B <= 0 || J <= 0 || H < 2 || W < 2 || !(radius > 0.f)) return fail(EPI_EINVAL, "bad shape or radius");
    if ((int)(radius + 0.5f) < 1) return fail(EPI_EINVAL, "radius must round to at least 1");
    cudaError_t e = epi::launch_peaks(heatmaps, locs, scores, B, J, H, W, radius, downsample, threshold, int_div,
                                      reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "peak kernel launch failed: %s", cudaGetErrorString(e));
    return EPI_OK;
}

int epi_find_peaks_best_f32(const float *heat, float *locs, float *scores, int32_t *src_index, int32_t S, int32_t B, int32_t J,
                            int32_t H, int32_t W, float radius, float downsample, float threshold, int32_t int_div, void *stream) {
    if (!heat || !locs || !scores) return fail(EPI_EINVAL, "null pointer");
    if (S <= 0 || B <= 0 || J <= 0 || H < 2 || W < 2 || !(radius > 0.f)) return fail(EPI_EINVAL, "bad shape or radius");
    if ((int)(radius + 0.5f) < 1) return fail(EPI_EINVAL, "radius must round to at least 1");
    if ((int64_t)B * J > INT32_MAX / 32) return fail(EPI_EINVAL, "B * J too large (one warp per joint, counted in int32)");
    cudaError_t e = epi::launch_peaks_best(heat, locs, scores, src_index, S, B, J, H, W, radius, downsample, threshold, int_div,
                                           reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(EPI_ECUDA, "peak kernel launch failed: %s", cudaGetErrorString(e));
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
