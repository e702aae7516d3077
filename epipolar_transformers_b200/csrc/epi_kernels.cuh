// epi_kernels.cuh — internal launch interface between the C ABI (epi_abi.cu) and the kernels.
#pragma once
#include <cuda_bf16.h>

#include "epi_common.cuh"

namespace epi {

// Host-side caches of per-device facts.  cudaFuncSetAttribute and the SM count concern the current device, so a host thread that
// runs the library on several devices keeps one entry per device; devices from kMaxDevices on are not cached (queried or set on
// every call).
constexpr int kMaxDevices = 64;
inline int current_device() {
    int dev = 0;
    return cudaGetDevice(&dev) == cudaSuccess ? dev : 0;
}

// one bit per device: whether a one-time setting (a kernel's shared-memory attribute) has been applied on that device
struct DeviceFlags {
    uint64_t bits = 0;
    bool has(int dev) const { return dev < kMaxDevices && ((bits >> dev) & 1u); }
    void set(int dev) { if (dev < kMaxDevices) bits |= 1ull << dev; }
};

// SMs of the current device, for persistent grids: queried once per host thread and device, 132 (an H100 SXM) if the query fails
inline int sm_count() {
    static thread_local int sms[kMaxDevices] = {};
    const int dev = current_device();
    int n = dev < kMaxDevices ? sms[dev] : 0;
    if (!n) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        if (dev < kMaxDevices) sms[dev] = n;
    }
    return n;
}

// Device-side view of one fused forward (built from EpiFusionParams by the ABI layer).
struct FusionArgs {
    const float *feat_ref;  int64_t ref_stride[4];   // fp32 (the caller's map, or a fp32 copy of a low-precision one) ...
    int ref_dtype;                            // ... except for the pipe kernel, which reads the caller's map in its own type (kF32/kBF16/kF16)
    const float *src_nhwc;                    // [N,H,W,C] contiguous, 16-byte aligned (zero-copy or staged) — warp kernel
    const __nv_bfloat16 *src_hi, *src_lo;     // [N,H,W,C] bf16 planes, src ≈ hi + lo — tile kernel
    const __nv_bfloat16 *ref_hi, *ref_lo;     // same for feat_ref — sector tiles and pipe kernel
                                              // (pipe kernel: lo planes are null for bf16 inputs, whose lo part is zero)
    const uint16_t *order;                    // [N,H*W] pixels sorted by epipolar angle — sector tiles only (else null)
    const float *P_ref, *P_src;
    const float *locs_in;
    float *out;             int64_t out_stride[4];
    __nv_bfloat16 *out_hi, *out_lo;           // optional: fused feature as bf16 (hi, lo) planes [N,H,W,C] (feeds the z GEMM)
    float *attn, *corr_pos, *locs_out;
    int N, C;                                 // N: pairs (S·N of the ABI)
    int n_ref, n_views;                       // pair n reads query item pair_items(n, n_ref, n_views[, vs]).q (feat_ref, ref_hi/lo, P_ref)
                                              // and source item .s (src planes / src_nhwc, P_src); n_views > 0: both are the V·n_ref view items
    float softmax_scale;
    int add_ref;
    int *tile_counter;                        // zeroed by the staging kernel; dynamic tile scheduler of the tile kernel
    const PairGeom *pair_geom;                // [N] per-pair constants (fp64-derived) written by the staging kernel — pipe kernel
    int *err_flag;                            // device word OR-ed with 1 when a work item had to be dropped (never for supported shapes)
    uint8_t *plan_cache;                      // optional persistent records of the pipe kernel's work items (camera-only data), or null
    int plan_records;                         // capacity of plan_cache in records of fusion_pipe_plan_record_bytes()
    const uint32_t *pair_epoch;               // [N] stride 32 words: epoch of each pair's cached plan (bumped by the staging kernel on a key miss)
    GeomCfg geom;
    int item_px;                              // pipe kernel: reference pixels per work item, 32 or 64 (fusion_pipe_item_pixels)
};

// Backward of the fused attention (epi_fusion_bwd.cu)
struct BwdArgs {
    const float *feat_ref;  int64_t ref_stride[4];
    const float *src_nhwc;                    // [N,H,W,C] contiguous fp32
    const float *P_ref, *P_src, *locs_in;
    const float *attn;                        // [N,K,H,W] saved by the forward
    const float *grad_out;  int64_t gout_stride[4];
    const float *grad_attn;                   // optional [N,K,H,W]
    float *grad_ref;        int64_t gref_stride[4];   // optional
    float *dsrc_nhwc;                         // optional [N,H,W,C] fp32, zero-initialised accumulator
    int N, C;
    float softmax_scale;
    int grad_keys, grad_vals;
    GeomCfg geom;
    // deterministic path (dsrc_nhwc unused): per-(pair, sample, pixel) scatter coefficients, the per-pair bound word (float bits,
    // zeroed, folded with atomicMax) and the zeroed [N,H,W,C] fixed-point accumulator of dL/dfeat_src
    float2 *coef;
    unsigned *pair_max;
    long long *acc;
};
cudaError_t launch_fusion_bwd(const BwdArgs &a, cudaStream_t st);
// deterministic backward: coefficient pass + fixed-point scatter into a.acc (a.coef, a.pair_max, a.acc set; a.dsrc_nhwc unused)
cudaError_t launch_fusion_bwd_det(const BwdArgs &a, cudaStream_t st, int &launched);
// fixed-point accumulator [N,HW,C] + per-pair bound words -> pixel-major fp32 dsrc (NaN for a pair whose bound is not finite)
cudaError_t launch_acc_to_f32(const long long *acc, const unsigned *pair_max, float *dsrc, int N, int HW, int C, cudaStream_t st);
// The views form of the backward: BwdArgs then describes a.N = V·S·N pairs on the V·n_ref items of one staged map.  Pair n reads
// feat_ref at its query item and src_nhwc at its source item (pair_items(n, n_ref, n_views, vs)), P_ref / P_src at the same
// items, and attn, grad_out, grad_attn and locs_in at n; grad_ref receives the pair's query term at n.  dsrc_nhwc, acc and
// pair_max are per source item (pair_max: the largest bound of the pairs that scatter into the item, det_item_scale).
struct BwdViews { int n_ref, n_views; ViewSources vs; };
cudaError_t launch_fusion_bwd_views(const BwdArgs &a, const BwdViews &vw, cudaStream_t st, bool det, int &launched);
// dL/dfeats of the views form, pixel-major fp32 [V·n_ref,HW,C]: for item i = v·n_ref + n, the query terms gq of its pairs
// (v·S + j)·n_ref + n summed in the order of j, plus its source term: dsrc[i] (float sums), or the fixed-point sums acc[i] with
// the item's bound word item_max[i], or nothing when both are null.  `g` may be `dsrc`.
cudaError_t launch_views_grad_sum(const float *gq, const float *dsrc, const long long *acc, const unsigned *item_max, float *g,
                                  const BwdViews &vw, int HW, int C, cudaStream_t st);

// z-projection epilogue:  y[n,o,p] = sum_c Wf[o,c]·x[n,c,p] + bf[o] (+x[n,o,p]) (+ref[n,o,p])
struct ZArgs {
    const float *x;         int64_t x_stride[4];     // pre-z fused feature
    const float *ref;       int64_t ref_stride[4];   // may be null; item n reads ref item pair_items(n, n_ref, n_views, vsrc).q
    void *y;                int64_t y_stride[4];     // element type: launch_z_epilogue's y_dtype
    const float *Wf, *bf;
    int N, C, HW, W, n_ref, n_views;
    int z_residual, add_ref;
    ViewSources vsrc;
};

// tensor-core z-projection: x arrives as bf16 (hi, lo) planes [N,H,W,C] written by the tile kernel
struct ZGemmArgs {
    const __nv_bfloat16 *x_hi, *x_lo;
    const __nv_bfloat16 *w_hi, *w_lo;         // Wf (+ I when ZRESIDUAL) [C out][C in] as bf16 (hi, lo) planes (written by the staging kernel)
    const float *Wf, *bf;
    const void *ref;        int64_t ref_stride[4];   // element type ref_dtype
    int ref_dtype;
    void *y;                int64_t y_stride[4];     // element type: launch_zgemm's y_dtype
    int N, C, HW, W, Npad, n_ref, n_views;    // item n reads ref item pair_items(n, n_ref, n_views, vs).q
    int z_residual, add_ref;
};
bool zgemm_supported(int C);
// vs: the views form's source table, the kernel's last parameter (behind the tensor maps); y_dtype (kF32 / kBF16 / kF16): element
// type of y, the fp32 result rounded once
cudaError_t launch_zgemm(const ZGemmArgs &z, const ViewSources &vs, int y_dtype, cudaStream_t st);

// vs: the views form's source table (vs.S = 0: none)
cudaError_t launch_fusion_warp(const FusionArgs &a, const ViewSources &vs, cudaStream_t st);
cudaError_t launch_fusion_tile(const FusionArgs &a, const ViewSources &vs, cudaStream_t st);
cudaError_t launch_fusion_pipe(const FusionArgs &a, const ViewSources &vs, cudaStream_t st);
bool fusion_pipe_shape_ok(int C, int H, int W, int K, bool has_locs_in);
size_t fusion_pipe_plan_record_bytes();
int fusion_pipe_item_pixels(int C, int H, int W);                  // 32 or 64
int fusion_pipe_plan_records(int N, int n_ref, int H, int W);   // N pairs on n_ref reference items
bool fusion_tile_shape_ok(int C, int H, int W, int K, bool has_locs_in);
// pair n: the cameras of pair_items(n, n_ref, n_views, vs)
cudaError_t launch_sector_order(const float *P_ref, const float *P_src, uint16_t *order, int N, int n_ref, int n_views,
                                const ViewSources &vs, const GeomCfg &gc, cudaStream_t st);
// `dtype` (kF32 / kBF16 / kF16): element type of the source map(s)
cudaError_t launch_split_planes(const void *src, const int64_t stride[4], __nv_bfloat16 *hi, __nv_bfloat16 *lo, int N, int C,
                                int H, int W, int *zero_me, int dtype, cudaStream_t st);

// planes: [ref_hi | ref_lo | src_hi | src_lo] for fp32 / fp16 maps, [ref_hi | src_hi] for bf16 maps (their lo part is zero);
// the reference planes hold n_ref items, the source planes (and the pair constants / orders) N pairs, pair n on reference n % n_ref;
// n_views > 0: `src` is null and only the reference planes are written, holding the n_views·n_ref view items (pair_items with vs);
// `launched`: kernels started on success (2 when a large map orders its pixels in a launch of its own)
cudaError_t launch_stage(const void *ref, const int64_t ref_stride[4], const void *src, const int64_t src_stride[4], int dtype,
                         __nv_bfloat16 *planes, const float *P_ref, const float *P_src, PairGeom *pair_geom, uint16_t *order,
                         float *order_key, const float *Wf, __nv_bfloat16 *w_planes, int w_add_identity, int *zero_words, int N, int n_ref,
                         int n_views, const ViewSources &vs, int C, int H, int W, const GeomCfg &gc, cudaStream_t st, int &launched);

cudaError_t launch_nchw_to_nhwc(const void *src, const int64_t stride[4], float *dst, int N, int C, int H, int W, int dtype,
                                cudaStream_t st);
// y_dtype (kF32 / kBF16 / kF16): element type of z.y, the fp32 result rounded once
cudaError_t launch_z_epilogue(const ZArgs &z, int y_dtype, cudaStream_t st);
// out_dtype (kF32 / kBF16 / kF16): fp32 sums rounded once (a gradient, or a 16-bit `out`); item n adds ref item
// pair_items(n, n_ref, n_views, vs).q of element type ref_dtype when ref is not null
cudaError_t launch_unstage(const float *pm, const void *ref, int ref_dtype, const int64_t ref_stride[4], void *out, int out_dtype,
                           const int64_t out_stride[4], int N, int n_ref, int n_views, const ViewSources &vs, int C, int H, int W,
                           cudaStream_t st);
// Heat-map epilogue (epi_head.cu): heat[n,j,p] = b[j] + Σ_c (A[j,c]·x[n,p,c] + B[j,c]·ref[q,c,p]), q = pair_items(n, n_ref,
// n_views, vs).q; x is the fused kernel's pixel-major fp32 plane [N,HW,C]; ref (element type ref_dtype, any strides) and B are
// null without the caller's residual.  1 <= J <= 64.
struct HeadArgs {
    const float *x;
    const void *ref;        int64_t ref_stride[4];
    int ref_dtype;
    const float *A, *B, *b;
    void *heat;             int64_t heat_stride[4];   // element type: launch_head's heat_dtype
    int N, C, HW, W, J, n_ref, n_views;
};
// heat_dtype (kF32 / kBF16 / kF16): element type of heat, the fp32 sum rounded once
cudaError_t launch_head(const HeadArgs &h, const ViewSources &vs, int heat_dtype, cudaStream_t st);
// A = Wh·(Wf + z_res·I) (Wh when Wf is null), b = Wh·bf + bh (null bh / bf: zero), fp64 sums rounded once; Wh [J,C], Wf [C,C]
cudaError_t launch_fold_head(const float *Wh, const float *bh, const float *Wf, const float *bf, int z_res, int J, int C, float *A,
                             float *b, cudaStream_t st);
cudaError_t launch_fold_z_bn(const float *zw, const float *zb, const float *g, const float *b, const float *mean,
                             const float *var, float eps, int C, float *wf, float *bf, cudaStream_t st);
cudaError_t launch_peaks(const float *heat, float *locs, float *scores, int B, int J, int H, int W, float radius, float downsample,
                         float threshold, int int_div, cudaStream_t st);
// heat [S,B,J,H,W]: per (b, j) the peak of the source with the highest score (first source on a tie); src_index may be null
cudaError_t launch_peaks_best(const float *heat, float *locs, float *scores, int *src_index, int S, int B, int J, int H, int W,
                              float radius, float downsample, float threshold, int int_div, cudaStream_t st);
// locs [V,N,J,2], scores [V,N,J], P [V,N,3,4] (float64 when P_f64, else float32) -> X [N,J,3], n_used [N,J]: one thread per (n, j)
cudaError_t launch_triangulate(const float *locs, const float *scores, const void *P, bool P_f64, double conf_thres, int V, int N,
                               int J, double *X, int *n_used, cudaStream_t st);
cudaError_t launch_sample_locs(const float *P_ref, const float *P_src, float *locs, int N, const GeomCfg &gc, cudaStream_t st);

// ---- recursive pictorial structure (epi_rpsm.cu) ----
constexpr int kRpsmMaxJoints = 32, kRpsmMaxNbins0 = 16, kRpsmMaxNbinsR = 4, kRpsmMaxDepth = 32;
// The tree and the level grids, built and checked on the host; passed by value.
struct RpsmTree {
    int J, E, root, max_depth;
    signed char parent[kRpsmMaxJoints];   // -1 at the root
    signed char edge[kRpsmMaxJoints];     // edge index of joint j as a child (the e-th non-root joint); -1 at the root
    signed char depth[kRpsmMaxJoints];
    signed char bfs[kRpsmMaxJoints];      // joints by ascending depth, the root first
};
struct RpsmArgs {
    const float *heat, *P, *crop, *root, *limb;   // [V,N,J,h,w], [V,N,3,4], [V,N,2,3], [N,3], [N,E]
    const uint32_t *mask;                         // level-0 pairwise, [E, B, ceil(B/32)], row = parent bin
    float *energy;                                // workspace: level-0 energies [N, J, B]
    int16_t *state;                               // workspace: level-0 arg-max states [N, E, B]
    float *pose;                                  // [N, J, 3]
    int V, N, h, w, n0, B, nr, depth, align;
    float img0, img1, tol;
    float g0[kRpsmMaxNbins0];                     // level-0 1-D grid (linspace), before the centre is added
    float gr[kRpsmMaxDepth][kRpsmMaxNbinsR];      // recursion r's 1-D grid
};
// launches: 1 unary + tree.max_depth max-product + 1 recursion kernel; returns the count in *launches
cudaError_t launch_rpsm(const RpsmArgs &a, const RpsmTree &t, cudaStream_t st, int *launches);
// packed [E, B, ceil(B/32)] bits: dense[e, p, k] != 0 (dense non-null), or |dist(X_p, X_k)| within tol of limb[e] on the
// level-0 grid g0 centred at the origin
cudaError_t launch_rpsm_pack(const float *dense, const float *limb, int E, int n0, const float *g0, float tol, uint32_t *packed,
                             cudaStream_t st);

}  // namespace epi
