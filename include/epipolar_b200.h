/* epipolar_b200.h — C ABI of the H100-native (sm_90a) epipolar-transformer fusion path (the names predate the H100 port).
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference has no FFI: its "operator" is the
 * Python call  Epipolar.forward(feat1, feat2, P1, P2, ...)  at
 *   /root/reference/modeling/layers/epipolar.py:82          (the forward being replaced)
 *   /root/reference/modeling/layers/epipolar.py:323-418     (grid2sample_locs — fused in-kernel)
 *   /root/reference/modeling/layers/epipolar.py:272-321     (epipolar_similarity — fused)
 *   /root/reference/modeling/layers/epipolar.py:248-255     (z conv + BN + residual — epilogue)
 *   /root/reference/vision/multiview.py:16-21,25-57,154-163 (camera_center / normalize /
 *                                                            de_normalize / pix2coord / coord2pix)
 *   /root/reference/modeling/backbones/resnet.py:385-388    (caller residual `ret + feat`)
 * A maintainer binds these symbols with ctypes (see INTEGRATION.md); the host side shipped
 * here (epipolar_transformers_b200/epipolar.py) does exactly that.
 *
 * Conventions: plain pointers + sizes, no torch types.  All tensor pointers are DEVICE
 * pointers to float32 unless a name ends in _host, except the feature maps feat_ref / feat_src and the backward's
 * grad_ref / grad_src, whose element type is the params' feat_dtype (EPI_DTYPE_*: float32, bfloat16 or float16; both maps
 * share it), and the forward's `out`, whose element type is the output dtype in bits 8-15 of feat_dtype (EPI_OUT_DTYPE;
 * float32 when they are zero).  Every other output stays float32.  The library never allocates persistent
 * device memory; the caller passes a workspace.  Every entry point is re-entrant, takes the
 * CUDA stream explicitly, never synchronises the device, and returns 0 on success or a
 * negative EPI_E* code (epi_last_error() gives a thread-local message).
 *
 * Alignment.  Every tensor pointer must be aligned to its element size.  Strides are in elements and may describe any
 * non-negative view: crops, channel slices, transposes, batch steps, and stride 0 on an input (a broadcast map).  Stricter:
 *   sample_locs_in, sample_locs_out, corr_pos   8 bytes (read and written as (x, y) float pairs): else EPI_EINVAL
 *   z_weight_folded                            16 bytes: else EPI_EINVAL
 *   workspace, cache                           256 bytes: else EPI_EINVAL
 * Nothing else is required: the library takes a 16-byte vector path only where it has checked the pointer and the strides
 * (e.g. an `out` that is not 16-byte aligned is written through a transposition pass instead of directly), so any other
 * alignment only costs speed.  Outputs must not overlap each other or the inputs.
 */
#ifndef EPIPOLAR_B200_H_
#define EPIPOLAR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EPI_ABI_VERSION 3

#define EPI_OK 0
#define EPI_EINVAL (-1)       /* bad argument / unsupported shape */
#define EPI_EWORKSPACE (-2)   /* workspace too small */
#define EPI_ECUDA (-3)        /* CUDA runtime error at launch (message has the cudaError string) */

/* element type of the feature maps (EpiFusionParams.feat_dtype, EpiFusionBwdParams.feat_dtype).  The result is the float32
 * computation applied to the exact input values: bfloat16 and float16 values are exact (hi, lo) bf16 pairs of the operand split. */
#define EPI_DTYPE_F32 0
#define EPI_DTYPE_BF16 1
#define EPI_DTYPE_F16 2
/* float64: only the cameras of epi_triangulate_dlt_f64 take it */
#define EPI_DTYPE_F64 3
/* element type of the forward's `out`, in bits 8-15 of EpiFusionParams.feat_dtype: feat_dtype = maps | EPI_OUT_DTYPE(out).
 * A bfloat16 or float16 `out` is the float32 result rounded once (to nearest even); attn, corr_pos and sample_locs_out stay
 * float32.  A library that predates the byte refuses a nonzero one with EPI_EINVAL ("unknown feat_dtype"). */
#define EPI_OUT_DTYPE(d) ((d) << 8)

/* kernel variants (EpiFusionParams.variant) */
#define EPI_VARIANT_AUTO 0    /* pipelined kernel when the shape allows, else sector / block tiles, else warp */
#define EPI_VARIANT_WARP 1    /* one warp per reference pixel, online softmax (baseline kernel) */
#define EPI_VARIANT_TILE 2    /* tensor-core kernel, 4x8 pixel tiles: shared-memory staged source taps, score interpolation */
#define EPI_VARIANT_SECTOR 3  /* tensor-core kernel, tiles of 32 pixels that share an epipolar line (sorted by epipolar angle) */
#define EPI_VARIANT_PIPE 4    /* warp-specialised, mbarrier-pipelined tensor-core kernel over epipolar-sector work items (default) */

typedef struct EpiFusionParams {
    /* ---- inputs ---------------------------------------------------------------------- */
    const void *feat_ref;         /* [N,C,H,W] logical, element type feat_dtype; element strides below (NCHW or channels-last) */
    int64_t ref_stride[4];
    const void *feat_src;         /* [N,C,H,W] logical, element type feat_dtype */
    int64_t src_stride[4];
    const float *P_ref;           /* [N,3,4] contiguous: KRT of the reference view  (forward arg P1) */
    const float *P_src;           /* [N,3,4] contiguous: KRT of the source view     (forward arg P2) */
    const float *sample_locs_in;  /* optional [K,N,H,W,2] contiguous, 8-byte aligned: normalised grid coords replacing the fused
                                     geometry (parity protocol T1: inject the reference's own locations) */
    /* ---- outputs --------------------------------------------------------------------- */
    float *out;                   /* [N,C,H,W] logical, strides below, element type EPI_OUT_DTYPE of feat_dtype (float32 unless
                                     bits 8-15 of feat_dtype say otherwise), aligned to its element size */
    int64_t out_stride[4];
    float *attn;                  /* optional [N,K,H,W] contiguous: softmax weights ("depth", epipolar.py:263) */
    float *corr_pos;              /* optional [N,H,W,2] contiguous, 8-byte aligned: arg-max correspondence, feature px (:237-242) */
    float *sample_locs_out;       /* optional [K,N,H,W,2] contiguous, 8-byte aligned: locations actually sampled (:183) */
    /* ---- optional folded eval-mode epilogue:  y = Wf·o + bf  (+ o if z_residual) ------ */
    const float *z_weight_folded; /* [C,C] row-major (out_ch, in_ch) = diag(gamma/sqrt(var+eps))·Wz, or NULL */
    const float *z_bias_folded;   /* [C] */
    /* ---- scratch ---------------------------------------------------------------------- */
    void *workspace;
    size_t workspace_bytes;       /* >= epi_fusion_workspace_bytes(p) */
    /* ---- shape & semantics ------------------------------------------------------------ */
    int32_t N, C, H, W, K;
    float downsample;             /* cfg.BACKBONE.DOWNSAMPLE */
    float img_scale;              /* cfg.DATASETS.IMAGE_RESIZE * PREDICT_RESIZE */
    float eps;                    /* 1e-3, epipolar.py:20 */
    float softmax_scale;          /* cfg.EPIPOLAR.SOFTMAXSCALE (0.125) */
    int32_t align_corners;        /* grid_sample semantics (torch>=1.3 default 0) */
    int32_t correct_normalize;    /* cfg.EPIPOLAR.USE_CORRECT_NORMALIZE */
    int32_t z_residual;           /* cfg.EPIPOLAR.ZRESIDUAL (only with z_weight_folded) */
    int32_t add_ref_residual;     /* 1: also add feat_ref (the caller's `ret + feat`, resnet.py:388) */
    int32_t variant;              /* EPI_VARIANT_* */
    int32_t feat_dtype;           /* bits 0-7: EPI_DTYPE_* of feat_ref and feat_src (ABI v3; 0 = float32).  bits 8-15:
                                     EPI_OUT_DTYPE(EPI_DTYPE_*) of `out` (0 = float32, the only output type before the byte).  Bits above 15 must
                                     be zero.  A 16-bit `out` always passes through an fp32 plane in the workspace, which the
                                     epilogue (z GEMM, fp32 z epilogue or transposition pass) rounds once; the workspace grows by
                                     that plane where the fused kernel would have stored `out` itself, and nothing else changes. */
    int32_t n_src;                /* source views per reference item, S = max(n_src, 1) (ABI v3; 0 or 1 = one source).  Pair
                                     p = s·N + n (0 <= s < S, 0 <= n < N) fuses reference item n with source item p:
                                     feat_ref / P_ref keep N items; feat_src is logical [S·N,C,H,W] (src_stride), P_src [S·N,3,4];
                                     out, attn, corr_pos have S·N items and sample_locs_in / sample_locs_out are [K,S·N,H,W,2].
                                     Every residual (add_ref_residual, also under the z epilogue) reads feat_ref[n]; z_residual
                                     adds pair p's own fused feature.  The reference map is staged once for all S sources.
                                     The cfg.EPIPOLAR.MULTITEST path of the reference (modeling/model.py:213-239) in one call. */
    union {
    int32_t reserved[1];          /* the name of this word before n_views (ABI v3 as first released) */
    int32_t n_views;              /* 0: the forms above.  V >= 2 (the views form; only where epi_fusion_views() returns 1): every view
                                     of a frame against every other, in one call.  feat_ref (ref_stride) is logical [V·N,C,H,W] and
                                     P_ref [V·N,3,4]: item v·N + n is view v of batch item n.  feat_src and P_src must be NULL and
                                     n_src 0 or 1; anything else (and n_views = 1 or < 0) is EPI_EINVAL.  Pair
                                     p = (v·(V−1) + j)·N + n (0 <= j < V−1) fuses query item v·N + n with source item u·N + n,
                                     u = j + (j >= v): the other views in increasing order.  out, attn, corr_pos have V·(V−1)·N items
                                     and sample_locs_in / sample_locs_out are [K,V·(V−1)·N,H,W,2].  Every residual reads the pair's
                                     query item.  Each pair's outputs are bit for bit those of a one-source call on (view v, view u);
                                     each view's map is staged once, as the query of V−1 pairs and the source of V−1 others. */
    };
    /* ---- optional persistent state (ABI v2) -------------------------------------------- */
    void *cache;                  /* device memory the caller keeps alive ACROSS calls and zero-fills once, or NULL.  Holds the
                                     per-pair constants and the epipolar pixel order keyed by (P_ref, P_src, H, W, downsample,
                                     img_scale): an unchanged camera pair skips their recomputation.  One cache per
                                     (module, device, stream); never share it between concurrently running calls. */
    size_t cache_bytes;           /* >= epi_fusion_cache_bytes(p) when cache != NULL */
} EpiFusionParams;

/* ABI version of the loaded library (== EPI_ABI_VERSION it was built with). */
int epi_version(void);

/* Thread-local description of the last error returned on this thread. */
const char *epi_last_error(void);

/* Bytes of scratch the forward needs for these shapes/strides/flags (0 is possible).  With n_src > 1 it covers N reference items
 * and S·N source items and pairs; with n_views = V, V·N view items and V·(V−1)·N pairs. */
size_t epi_fusion_workspace_bytes(const EpiFusionParams *p);

/* Bytes of the optional persistent cache for these shapes (0 when the selected kernel keeps no cross-call state); S·N pairs, or
 * V·(V−1)·N with n_views = V. */
size_t epi_fusion_cache_bytes(const EpiFusionParams *p);

/* The fused forward: geometry + K bilinear taps + softmax(QK)·V (+ z/BN epilogue, + residuals).
 * Replaces Epipolar.forward for ATTENTION='avg', SIMILARITY='dot', SOFTMAX_ENABLED.
 * Asynchronous on `stream` (a cudaStream_t); returns launch-time errors only. */
int epi_fusion_forward_f32(const EpiFusionParams *p, void *stream);

/* ---- backward of the fused attention (SURVEY.md 8f rank 1) --------------------------------------------------------
 * Replaces autograd through  F.grid_sample x2 / mul / sum / softmax  of /root/reference/modeling/layers/epipolar.py:188-247
 * (called under autograd by /root/reference/engine/trainer.py:72).  Sample locations are constants (:178 torch.no_grad).
 * grad_keys / grad_vals select the OTHER_GRAD members 'other1' / 'other2' (:141-153).  The z conv + BN of training mode
 * stay in PyTorch, so `grad_out` is the gradient w.r.t. the PRE-z fused feature. */
typedef struct EpiFusionBwdParams {
    const void *feat_ref;         /* [N,C,H,W] logical, element type feat_dtype, strides below */
    int64_t ref_stride[4];
    const void *feat_src;         /* element type feat_dtype */
    int64_t src_stride[4];
    const float *P_ref, *P_src;   /* [N,3,4] */
    const float *sample_locs_in;  /* optional, as in the forward (contiguous, 8-byte aligned) */
    const float *attn;            /* [N,K,H,W] contiguous: the forward's attention output */
    const float *grad_out;        /* [N,C,H,W] logical: dL/d(fused feature) */
    int64_t gout_stride[4];
    const float *grad_attn;       /* optional [N,K,H,W] contiguous: dL/d(attention output) */
    void *grad_ref;               /* optional out [N,C,H,W] logical, element type feat_dtype: dL/dfeat_ref (fp32, rounded once) */
    int64_t gref_stride[4];
    void *grad_src;               /* optional out [N,C,H,W] logical, element type feat_dtype: dL/dfeat_src (overwritten, not accumulated) */
    int64_t gsrc_stride[4];
    void *workspace;
    size_t workspace_bytes;       /* >= epi_fusion_backward_workspace_bytes(p) */
    int32_t N, C, H, W, K;
    float downsample, img_scale, eps, softmax_scale;
    int32_t align_corners, correct_normalize;
    int32_t grad_keys, grad_vals; /* 'other1' / 'other2' in cfg.EPIPOLAR.OTHER_GRAD */
    int32_t feat_dtype;           /* EPI_DTYPE_* of feat_ref, feat_src, grad_ref and grad_src (ABI v3; 0 = float32) */
    int32_t deterministic;        /* 0: dL/dfeat_src is summed with float atomics, whose order (and so last bits) varies from run to
                                     run.  1: bit-reproducible: the same inputs give the same bits, whatever the batch around a
                                     pair and the layouts; sums in per-pair int64 fixed point (DESIGN.md §5), more workspace and two
                                     more launches.  A pair whose gradients or maps hold a NaN or inf gets an all-NaN dL/dfeat_src.
                                     dL/dfeat_ref is order-fixed on both paths and the same bits on both.  Other values: EPI_EINVAL. */
    int32_t reserved[2];
} EpiFusionBwdParams;

size_t epi_fusion_backward_workspace_bytes(const EpiFusionBwdParams *p);
int epi_fusion_backward_f32(const EpiFusionBwdParams *p, void *stream);
/* 1: this library honours EpiFusionBwdParams.deterministic (a library built before the field read it as a reserved word). */
int epi_fusion_backward_deterministic(void);
/* 1: this library honours EpiFusionParams.n_views (a library built before the field read it as a reserved word and would run a
 * one-source call). */
int epi_fusion_views(void);

/* ---- the views form with a caller's source table --------------------------------------------------------------------------
 * The views form (n_views = V >= 2, see EpiFusionParams.n_views) with the sources chosen by the caller instead of every other
 * view: view v of item n is fused with views sources_host[v·S + j], 0 <= j < S.  sources_host is a [V][S] int32 table in HOST
 * memory, read and checked during the call (the caller may reuse it once the call returns).  It reaches the kernels inside their
 * launch parameters, so the call neither synchronises nor copies from pageable memory; that bounds the table to
 * V·S <= EPI_VIEW_SOURCES_MAX entries.  Every other field of p means what it means in the views form (feat_src and P_src NULL,
 * n_src 0 or 1).  Pair p = (v·S + j)·N + n fuses query item v·N + n with source item sources_host[v·S + j]·N + n.  out, attn and
 * corr_pos have V·S·N items, sample_locs_in / sample_locs_out are [K,V·S·N,H,W,2], and every residual reads the pair's query
 * item.  Each pair's outputs (every output and epilogue, every variant and feat_dtype, injected locations, with or without the
 * cache) are bit for bit those of a one-source call on (view v, view u) at item n; each view's map is staged once.  The cache
 * stays keyed per pair by that pair's cameras, so a changed table on the same cache gives fresh-call results.
 * Duplicate entries are allowed.  EPI_EINVAL (with a message) for a NULL table, S < 1, n_views < 2, V·S > EPI_VIEW_SOURCES_MAX,
 * an entry outside [0, V), an entry equal to its own view (a self-pair), V·S·N > 65535 pairs, and every refusal of the views form.
 * Its backward is epi_fusion_views_backward_f32 below. */
#define EPI_VIEW_SOURCES_MAX 256
int epi_fusion_view_sources_forward_f32(const EpiFusionParams *p, const int32_t *sources_host, int32_t S, void *stream);
/* Workspace / cache bytes of that call: V·N staged view items and V·S·N pairs.  0 when the table or params cannot be planned. */
size_t epi_fusion_view_sources_workspace_bytes(const EpiFusionParams *p, const int32_t *sources_host, int32_t S);
size_t epi_fusion_view_sources_cache_bytes(const EpiFusionParams *p, const int32_t *sources_host, int32_t S);
/* 1: this library has the source-table entry points above (a library built before them lacks this symbol). */
int epi_fusion_view_sources(void);

/* ---- backward of the views form ---------------------------------------------------------------------------------------------
 * The gradient of every view item of a frame, for the pairs of the views form (n_views = V, sources_host a [V][S] host table
 * read as in epi_fusion_view_sources_forward_f32, or NULL with S = 0 for every other view, S = V−1).  Pair p = (v·S + j)·N + n
 * fuses query item v·N + n with source item u·N + n, u = sources_host[v·S + j] (or j + (j >= v)).  Fields of p:
 *   N                          items per view;
 *   feat_ref / ref_stride      the V·N view maps [V·N,C,H,W] (feat_dtype), P_ref [V·N,3,4] (or sample_locs_in);
 *   attn, grad_out, grad_attn, sample_locs_in    per pair: [V·S·N,K,H,W], [V·S·N,C,H,W], [V·S·N,K,H,W], [K,V·S·N,H,W,2];
 *   grad_ref / gref_stride     out [V·N,C,H,W] (feat_dtype, the caller's strides), overwritten with
 *                              dL/dfeats[i] = Σ over pairs p with query item i of dL/dfeat_ref(p)
 *                                           + Σ over pairs p with source item i of dL/dfeat_src(p)   (grad_keys / grad_vals select
 *                              the source terms, as in epi_fusion_backward_f32; with both 0 only the query terms remain);
 *   feat_src, P_src, grad_src  must be NULL.
 * Every term is what epi_fusion_backward_f32 computes for pair p; the sums are formed in fp32 and rounded once.  Each view map is
 * staged once.  deterministic = 1: bit-reproducible, the source terms summed in int64 fixed point per item, with a scale set by
 * the bounds of that item's pairs (so by its frame alone); an item one of whose pairs has a non-finite bound gets all NaN.  The
 * query terms are summed in pair order on both paths.  EPI_EINVAL (with a message) for every refusal of epi_fusion_backward_f32,
 * every table refusal of epi_fusion_view_sources_forward_f32, n_views < 2, more than 65535 pairs and a non-NULL
 * feat_src / P_src / grad_src. */
int epi_fusion_views_backward_f32(const EpiFusionBwdParams *p, int32_t n_views, const int32_t *sources_host, int32_t S, void *stream);
/* Workspace bytes of that call (0 when the table or params cannot be planned). */
size_t epi_fusion_views_backward_workspace_bytes(const EpiFusionBwdParams *p, int32_t n_views, const int32_t *sources_host, int32_t S);
/* 1: this library has the views backward above (a library built before it lacks this symbol). */
int epi_fusion_views_backward(void);

/* ---- heat-maps: the pose head's 1×1 conv as the forward's epilogue ------------------------------------------------------
 * The eval step of the pose network after the fusion layer is  final_layer(ret + feat)  (/root/reference/modeling/backbones/
 * resnet.py:388,421).  With X the pre-z fused feature, (Wf, bf) the z / BN fold (epi_fold_z_bn_f32), R the caller's residual
 * feat_ref of the pair's query item and (Wh [J,C], bh [J]) the head:
 *   heat = Wh·(Wf·X + bf + z_res·X + R) + bh = A·X + B·R + b,   A = Wh·(Wf + z_res·I),  B = Wh,  b = Wh·bf + bh
 * (without z: A = Wh, b = bh; without the caller's residual: B = 0).  The fused feature is never written to `out`. */
typedef struct EpiHeadParams {
    const float *A;               /* [J,C] row-major, 4-byte aligned (epi_fold_head_f32) */
    const float *B;               /* [J,C] row-major: the head weight Wh, adding the caller's residual feat_ref; or NULL (none) */
    const float *b;               /* [J] */
    void *heat;                   /* [pairs,J,H,W] logical, any element strides below, element type EPI_OUT_DTYPE of feat_dtype
                                     (float32 unless bits 8-15 of feat_dtype say otherwise), aligned to its element size */
    int64_t heat_stride[4];
    int32_t J;                    /* joints, 1 <= J <= 64 */
    int32_t reserved[3];          /* must be zero */
} EpiHeadParams;

/* Fold z / BN and the head into (A, b) of EpiHeadParams on the device: A = Wh·(Wf + z_residual·I), b = Wh·bf + bh, each element
 * summed in fp64 and rounded once to fp32.  Wh [J,C] row-major; bh [J] or NULL (zero); Wf [C,C] (epi_fold_z_bn_f32) or NULL
 * (A = Wh, b = bh: a layer without z); bf [C] or NULL (zero).  A_out [J,C], b_out [J].  One launch; never synchronises, so it
 * can be captured in a CUDA graph.  EPI_EINVAL for a NULL Wh / A_out / b_out, J < 1 or C < 1. */
int epi_fold_head_f32(const float *Wh, const float *bh, const float *Wf, const float *bf, int32_t z_residual, int32_t J, int32_t C,
                      float *A_out, float *b_out, void *stream);

/* The forward of any form (pair, n_src, n_views, or the views form with a source table: sources_host a [V][S] host table as in
 * epi_fusion_view_sources_forward_f32, or NULL with S = 0 for none) with the head as its epilogue: h->heat receives, per pair,
 * A·X + B·R + b; attn, corr_pos and sample_locs_out are what the same call without the head writes, bit for bit.  The fused kernel
 * stores X as an fp32 pixel-major plane in the workspace, and one more launch applies the head: every heat element is an fp32 sum
 * over c = 0 .. C−1 in one fixed order (b, then A[j,c]·X[c] and B[j,c]·R[c] for increasing c), so each pair's heat is bit for bit
 * that of the pair-form call on that pair, and a 16-bit heat is the fp32 heat rounded once.  EPI_EINVAL (with a message) for a
 * non-NULL out, z_weight_folded or nonzero add_ref_residual (A, B and b express them), a NULL h / A / b / heat, J < 1 or J > 64,
 * nonzero reserved words, and every refusal of the form it runs. */
int epi_fusion_heatmaps_f32(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S, void *stream);
/* Workspace / cache bytes of that call (0 when the params, the head or the table cannot be planned). */
size_t epi_fusion_heatmaps_workspace_bytes(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S);
size_t epi_fusion_heatmaps_cache_bytes(const EpiFusionParams *p, const EpiHeadParams *h, const int32_t *sources_host, int32_t S);
/* 1: this library has the heat-map entry points above (a library built before them lacks this symbol). */
int epi_fusion_heatmaps(void);

/* Only the geometry: sample locations [K,N,H,W,2] for (P_ref,P_src)  (grid2sample_locs). */
int epi_sample_locs_f32(const float *P_ref, const float *P_src, float *sample_locs_out, int32_t N,
                        int32_t H, int32_t W, int32_t K, float downsample, float img_scale, float eps,
                        int32_t correct_normalize, void *stream);

/* find_tensor_peak_batch for a whole batch (replaces the per-item Python loop at
 * /root/reference/modeling/backbones/resnet.py:423-428 over modeling/backbones/basic_batch.py:17-63):
 * heatmaps [B,J,H,W] contiguous -> locs [B,J,2] (x, y in image coordinates, pix2coord applied) and scores [B,J].
 * radius = cfg.KEYPOINT.SIGMA; threshold 1e-6 in the reference; int_div = 1 reproduces torch < 1.4's integer `index / W`,
 * 0 the true division of current torch (what the reference computes under the torch installed with this library).
 * Non-finite values follow torch: the arg-max is the first NaN if the map holds one, else the first maximum; the threshold
 * zeroes values <= threshold and keeps NaN, so a NaN or a zero bilinear weight times ±inf in the window gives a NaN location.
 * EPI_EINVAL for a radius that is not finite and > 0, one whose R = int(radius + 0.5) is outside 1 .. EPI_PEAKS_MAX_R (the
 * (2R+1)^2-sample window is counted in int32), or B·J > INT32_MAX / 32 (one warp per joint, counted in int32). */
#define EPI_PEAKS_MAX_R 23169
int epi_find_peaks_f32(const float *heatmaps, float *locs, float *scores, int32_t B, int32_t J, int32_t H, int32_t W,
                       float radius, float downsample, float threshold, int32_t int_div, void *stream);

/* The best-source selection of the reference's multi-view test (modeling/model.py:229-234: torch.max over the sources' peak
 * scores, then gather of their locations): heat [S,B,J,H,W] contiguous -> for every (b, j) the peak of the source with the
 * highest score, locs [B,J,2], scores [B,J] and optionally (src_index != NULL) that source's index [B,J] as int32.  Each source's
 * peak is computed exactly as epi_find_peaks_f32 computes it, with the same refusals; as torch.max, the first source with a NaN
 * score wins, else the first with the highest score.  S = 1 returns epi_find_peaks_f32's result bit for bit. */
int epi_find_peaks_best_f32(const float *heat, float *locs, float *scores, int32_t *src_index, int32_t S, int32_t B, int32_t J,
                            int32_t H, int32_t W, float radius, float downsample, float threshold, int32_t int_div, void *stream);

/* Linear (DLT) triangulation of every (frame, joint) in one launch: the reference's KEYPOINT.TRIANGULATION = 'pymvg' mode
 * (vision/triangulation.py, triangulate_pymvg, and pymvg's find3d, with zero distortion).  For the problem (n, j):
 *   1. views: t = conf_thres in fp64; repeat { sel = {v : scores[v,n,j] > (float)t}; stop if t < -1; if |sel| <= 1,
 *      t = t - 0.05 (fp64) and repeat; else stop }.  The compare is float32, as numpy compares a float32 array with a Python
 *      float; a NaN score is never selected.
 *   2. A: per selected view, in increasing view order, the rows x·M[2] - M[0] and y·M[2] - M[1] in fp64, M = P[v,n], (x, y) =
 *      locs[v,n,j].
 *   3. X[n,j] = w[:3] / w[3], w the right singular vector of A's smallest singular value (Givens QR of A's rows into a 4x4 R,
 *      then one-sided Jacobi on R, all in fp64; AᵀA is never formed).
 * n_used[n,j] = |sel| (0 .. V).  X is NaN when |sel| < 2 or a selected view has a non-finite location or camera entry;
 * w[3] = 0 gives the IEEE quotient.  locs [V,N,J,2] (image px, any resizing already applied), scores [V,N,J] and P [V,N,3,4] are
 * contiguous; P is float32 (P_dtype = EPI_DTYPE_F32) or float64 (EPI_DTYPE_F64).  One launch on `stream`; never synchronises,
 * so it can be captured in a CUDA graph.  EPI_EINVAL (with a message) for a NULL pointer, V < 2 or V > 64, N < 1, J < 1,
 * N·J > 2^31 - 1, an unknown P_dtype, a non-finite conf_thres or one above 1000 (step 1 would count down from it for
 * (conf_thres + 1) / 0.05 passes), and locs, X or a float64 P not 8-byte aligned or scores, n_used or a float32 P not 4-byte
 * aligned. */
int epi_triangulate_dlt_f64(const float *locs, const float *scores, const void *P, int32_t P_dtype, double conf_thres, int32_t V,
                            int32_t N, int32_t J, double *X, int32_t *n_used, void *stream);
/* 1: this library has epi_triangulate_dlt_f64 (a library built before it lacks this symbol). */
int epi_triangulate(void);

/* The reference's recursive pictorial-structure model (KEYPOINT.TRIANGULATION = 'rpsm', modeling/pictorial_cuda.py) for N
 * frames at once.  The tree is the host array parents[J] (the root -1, every other joint its parent's index); a joint's
 * children are taken in ascending index, and edge e is the e-th non-root joint (limb_length's and the mask's edge order).
 * Level 0 is a cube of first_nbins^3 = B bins of side grid_size around root[n], one grid for all joints, its pairwise term the
 * caller's packed 0/1 mask; recursion r = 1..recur_depth puts recur_nbins^3 bins of side grid_size / first_nbins /
 * recur_nbins^(r-1) around each joint's current estimate, its pairwise term |dist + 1e-9 - limb_length| < tolerance.  The
 * arithmetic, operation by operation, is in csrc/epi_rpsm.cu's header; the pose is the chosen bins' float32 coordinates. */
typedef struct EpiRpsmParams {
    const float *heat;          /* [V,N,J,h,w] heat-maps */
    const float *P;             /* [V,N,3,4] original-image cameras (origK @ RT) */
    const float *crop;          /* [V,N,2,3] crop affine of each view (get_affine_transform(center, scale, 0, image_size)) */
    const float *root;          /* [N,3] centre of the level-0 cube */
    const float *limb_length;   /* [N,E] limb lengths (E = J - 1), used by the recursions */
    const uint32_t *pairwise;   /* [E,B,ceil(B/32)] level-0 mask, bit k of row p = parent bin p may take child bin k */
    const int32_t *parents;     /* HOST array [J] */
    float *pose;                /* [N,J,3] output */
    void *workspace;            /* epi_rpsm_workspace_bytes(), 256-byte aligned */
    size_t workspace_bytes;
    int32_t V, N, J, h, w;
    int32_t first_nbins, recur_nbins, recur_depth, align_corners;
    float image_size[2];        /* IMAGE_SIZE (x, y) in pixels */
    double grid_size;           /* GRID_SIZE (mm); the level sizes are divided in fp64 */
    double tolerance;           /* LIMB_LENGTH_TOLERANCE (mm), compared in float32 */
} EpiRpsmParams;

/* Bytes of workspace for `p`: the level-0 energies (N·J·B float32) and arg-max states (N·E·B int16). */
size_t epi_rpsm_workspace_bytes(const EpiRpsmParams *p);
/* pose for every frame; 2 + (the tree's depth) launches on `stream` whatever N is (epi_last_launch_count()); never
 * synchronises, so it can be captured in a CUDA graph.  EPI_EINVAL (with a message) for a NULL pointer, V outside [2, 64],
 * N < 1, J outside [1, 32] or a parents array that is not one tree, first_nbins outside [2, 16], recur_nbins outside [2, 4],
 * recur_depth outside [0, 32], h or w < 2, a non-finite or non-positive grid_size, tolerance or image size, a float pointer
 * not 4-byte aligned, a workspace not 256-byte aligned or smaller than epi_rpsm_workspace_bytes(). */
int epi_rpsm_f32(const EpiRpsmParams *p, void *stream);
/* The packed level-0 mask [E, B, ceil(B/32)] (B = nbins^3, bits past B zero) on the device, from either a dense [E,B,B]
 * float32 mask (bit = entry != 0; limb_length NULL) or limb lengths [E] (dense NULL) on the level-0 grid centred at the
 * origin, with the recursions' rule |dist + 1e-9 - limb_length| < tolerance.  One launch on `stream`.  EPI_EINVAL for both or
 * neither source, a NULL or misaligned packed, E outside [0, 31], nbins outside [2, 16], a non-finite or non-positive
 * grid_size or (limb lengths) tolerance. */
int epi_rpsm_pairwise_pack(const float *dense, const float *limb_length, int32_t E, int32_t nbins, double grid_size,
                           double tolerance, uint32_t *packed, void *stream);
/* 1: this library has the epi_rpsm_* entry points (a library built before them lacks this symbol). */
int epi_rpsm(void);

/* Fold conv1x1 z + eval BatchNorm into (Wf, bf) on the device, no host sync:
 *   Wf[o,c] = s[o]·Wz[o,c],  bf[o] = s[o]·(bz[o] − mean[o]) + beta[o],  s = gamma/sqrt(var+bn_eps). */
int epi_fold_z_bn_f32(const float *z_weight, const float *z_bias, const float *bn_weight,
                      const float *bn_bias, const float *bn_mean, const float *bn_var, float bn_eps,
                      int32_t C, float *w_folded, float *b_folded, void *stream);

/* Diagnostic: one-CTA wgmma GEMM in the exact operand forms the fusion kernels use
 * (mode 0: D[128,N] = A[128,K]·B[N,K]^T, both K-major;  mode 1: D[128,N] = At[K,128]^T·B[N,K]^T, A MN-major;
 * split=1: bf16 (hi,lo) three-term products).  All pointers device fp32, row-major. */
int epi_umma_selftest(int mode, const float *A, const float *B, float *D, int N, int K, int split, void *stream);

/* Measurement aid (bench.py roofline): when enabled on this thread, epi_fusion_forward_f32 brackets its dominant
 * kernel (the fused attention kernel) with CUDA events on the caller's stream; epi_kernel_timing_last_ms()
 * synchronises on them and returns that launch's duration in milliseconds (< 0 if there is none). */
int epi_kernel_timing_enable(int on);
float epi_kernel_timing_last_ms(void);
/* same, per launch group: ms3[0] operand staging, ms3[1] fused attention kernel, ms3[2] epilogue pass */
int epi_kernel_timing_last3(float *ms3);

/* Number of kernels the last successful forward or backward call on this thread launched. */
int epi_last_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* EPIPOLAR_B200_H_ */
