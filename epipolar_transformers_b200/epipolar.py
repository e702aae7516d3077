"""Host side of the CUDA epipolar fusion path: `Epipolar(nn.Module)` with the reference's
constructor / forward contract, calling the C ABI (include/epipolar_b200.h) through ctypes.

Mirrors /root/reference/modeling/layers/epipolar.py:
  Epipolar.__init__  :12-80   (cfg keys, parameter names z.* / bn.* kept for checkpoints)
  Epipolar.forward   :82-269  (signature, 4-tuple return contract :262-269)
and the caller residual of /root/reference/modeling/backbones/resnet.py:377-388
(`fused_other_feat`).  PyTorch is used here only for device memory, streams and parameters;
every arithmetic step of the graded path runs in libepipolar_b200.so.  No CPU fallback.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np
import torch
from torch import nn

from . import _lib
from .config import get_global_cfg
from .peaks import find_tensor_peak_batch, find_tensor_peak_best

_EPSILON = 0.001          # epipolar.py:20


class ZeroInitBN(nn.BatchNorm2d):
    """BatchNorm2d whose affine weight AND bias start at zero (reference: modeling/layers/BN.py:48-52);
    state-dict keys identical to the reference's zeroinitBN."""

    def reset_parameters(self):
        super().reset_parameters()
        if self.affine:
            nn.init.zeros_(self.weight)
            nn.init.zeros_(self.bias)


def _strides4(t: torch.Tensor):
    return (ctypes.c_int64 * 4)(*t.stride())


def _aligned_locs(t: torch.Tensor) -> torch.Tensor:
    """sample locations as the ABI takes them: contiguous float32 on the device, 8-byte aligned (the kernels load (x, y) as one
    pair).  `.contiguous()` keeps a contiguous view that starts at an odd element, so such a view is copied."""
    t = t.contiguous()
    return t if t.data_ptr() % 8 == 0 else t.clone()


# element types the kernels read natively (EPI_DTYPE_*); bf16 / fp16 maps give the fp32 result of their exact values
FEAT_DTYPES = {torch.float32: _lib.EPI_DTYPE_F32, torch.bfloat16: _lib.EPI_DTYPE_BF16, torch.float16: _lib.EPI_DTYPE_F16}
_DTYPE_NAMES = {torch.float32: "float32", torch.bfloat16: "bfloat16", torch.float16: "float16"}


def _check_feat_pair(feat_ref, feat_src, out=None, out_dtype=torch.float32):
    """Both maps: 4-D, one supported dtype, on the GPU; `out_dtype` float32, bfloat16 or float16, and a caller-supplied `out` of
    that dtype.  -> EPI_DTYPE_* code of the maps."""
    if out_dtype not in FEAT_DTYPES:
        raise TypeError("out_dtype must be torch.float32, torch.bfloat16 or torch.float16 (got %r)" % (out_dtype,))
    for name, t in (("feat_ref", feat_ref), ("feat_src", feat_src)):
        if not isinstance(t, torch.Tensor) or t.dim() != 4:
            raise ValueError("%s must be a 4-D tensor [N,C,H,W]" % name)
        if t.dtype not in FEAT_DTYPES:
            raise TypeError("%s must be float32, bfloat16 or float16 (got %s)" % (name, t.dtype))
    if feat_ref.dtype != feat_src.dtype:
        raise TypeError("feat_ref and feat_src must have the same dtype (got %s and %s)" % (feat_ref.dtype, feat_src.dtype))
    if out is not None and out.dtype != out_dtype:
        if out_dtype == torch.float32:
            raise TypeError("out must be float32 (got %s): the fused feature is computed and stored in float32, unless "
                            "out_dtype asks for bfloat16 or float16" % out.dtype)
        raise TypeError("out must be %s (got %s): out_dtype=%s" % (_DTYPE_NAMES[out_dtype], out.dtype, out_dtype))
    for name, t in (("feat_ref", feat_ref), ("feat_src", feat_src)):
        if not t.is_cuda:
            raise RuntimeError("%s is on %s: the CUDA epipolar path has no CPU implementation" % (name, t.device))
    return FEAT_DTYPES[feat_ref.dtype]


class FusionState:
    """Persistent scratch of one caller (module) on one device: the workspace, the cross-call cache of the C ABI
    (pixel order + pair constants keyed by the camera matrices) and the prepared parameter block.  Re-using it removes
    the per-call allocations and lets an unchanged camera pair skip its setup work.  A state must not be shared by
    calls that can run concurrently (different streams / threads): give each its own."""

    __slots__ = ("key", "ws", "cache", "params")

    def __init__(self):
        self.key = None
        self.ws = None
        self.cache = None
        self.params = None


def epipolar_fusion(feat_ref, feat_src, P_ref, P_src, *, K, downsample=4.0, img_scale=1.0,
                    softmax_scale=0.125, correct_normalize=False, align_corners=False,
                    z_folded=None, z_residual=False, add_ref_residual=False,
                    sample_locs_in=None, want_attn=True, want_corr=True, want_locs=False,
                    variant="auto", out=None, state: Optional[FusionState] = None, out_dtype=torch.float32, head=None):
    """Functional form of the fused forward.  Returns (out, corr_pos|None, attn|None, sample_locs|None).

    feat_ref/feat_src: CUDA [N,C,H,W] (NCHW or channels_last strides), both float32, both bfloat16 or both float16 (what a
      backbone under torch.autocast produces).  The result is the float32 computation on the exact input values.
    out_dtype: dtype of `out` (and of a caller-supplied `out`): float32, or bfloat16 / float16, the float32 result rounded
      once to nearest even (for a model cast to half precision).  corr_pos, attn and sample_locs are float32.
    P_ref/P_src: [N,3,4] (cast to float32 like modeling/model.py:183-195).
    z_folded: optional (Wf [C,C], bf [C]) from `fold_z_bn` (eval-mode epilogue, epipolar.py:249-253).
    sample_locs_in: optional [K,N,H,W,2] normalised locations replacing the fused geometry.
    state: optional FusionState (persistent workspace + camera-keyed cache); without it scratch is allocated per call.
    head: optional (weight [J,C] or [J,C,1,1], bias [J] | None), the pose head's 1x1 conv (`final_layer`), or that conv itself,
      1 <= J <= 64: the call returns (heat [N,J,H,W], corr_pos, attn, sample_locs) with heat = head(z/BN epilogue(fused) +
      feat_ref if add_ref_residual), of dtype out_dtype, and the fused feature is never stored (`out` must be None).  corr_pos,
      attn and sample_locs are bit for bit those of the call without a head.  Inference only (`fold_head`, DESIGN.md §3.7).
    """
    lib = _lib.load()
    if head is not None:
        _lib.require_heatmaps(lib)
    dcode = _check_feat_pair(feat_ref, feat_src, out, out_dtype)
    if feat_ref.shape != feat_src.shape or feat_ref.device != feat_src.device:
        raise ValueError("feat_ref and feat_src must have the same shape and device")
    hp = None if head is None else _head_operands(lib, head, feat_ref, feat_src, out, z_folded, z_residual, add_ref_residual)
    return _fusion(lib, dcode, 1, feat_ref, feat_src, P_ref, P_src, K=K, downsample=downsample, img_scale=img_scale,
                   softmax_scale=softmax_scale, correct_normalize=correct_normalize, align_corners=align_corners,
                   z_folded=None if hp else z_folded, z_residual=z_residual and not hp,
                   add_ref_residual=add_ref_residual and not hp, sample_locs_in=sample_locs_in,
                   want_attn=want_attn, want_corr=want_corr, want_locs=want_locs, variant=variant, out=out, state=state,
                   out_dtype=out_dtype, head=hp)


def epipolar_fusion_multi(feat_ref, feat_srcs, P_ref, P_srcs, *, K, downsample=4.0, img_scale=1.0,
                          softmax_scale=0.125, correct_normalize=False, align_corners=False,
                          z_folded=None, z_residual=False, add_ref_residual=False,
                          sample_locs_in=None, want_attn=True, want_corr=True, want_locs=False,
                          variant="auto", out=None, state: Optional[FusionState] = None, out_dtype=torch.float32,
                          head=None):
    """Fuses every reference item with S source views in one call: the multi-view test path of the reference
    (cfg.EPIPOLAR.MULTITEST, modeling/model.py:213-239), where each reference batch is fused against every other view.
    Source s of item n gives exactly what `epipolar_fusion(feat_ref, feat_srcs[s], P_ref, P_srcs[s])` gives, but the
    reference map is staged once and the S pairs share one launch chain.

    feat_ref: [N,C,H,W] as in `epipolar_fusion`; feat_srcs: [S,N,C,H,W], or a sequence of S [N,C,H,W] maps (stacked);
    P_ref: [N,3,4]; P_srcs: [S,N,3,4]; sample_locs_in: optional [K,S,N,H,W,2]; out: optional [S,N,C,H,W] of dtype out_dtype
    (float32, or bfloat16 / float16 as in `epipolar_fusion`).
    Every residual (add_ref_residual, also under z) adds feat_ref[n].  Returns
    (out [S,N,C,H,W], corr_pos [S,N,H,W,2] | None, attn [S,N,K,H,W] | None, sample_locs [K,S,N,H,W,2] | None); with a `head`
    (as in `epipolar_fusion`) heat [S,N,J,H,W] in place of out.
    Inference only (no backward for several sources): inputs that require grad under grad mode raise RuntimeError."""
    lib = _lib.load()
    if head is not None:
        _lib.require_heatmaps(lib)
    if isinstance(feat_srcs, (list, tuple)):
        if not feat_srcs or not all(isinstance(t, torch.Tensor) for t in feat_srcs):
            raise ValueError("feat_srcs must be a [S,N,C,H,W] tensor or a non-empty sequence of [N,C,H,W] tensors")
        if len({(tuple(t.shape), t.dtype, t.device) for t in feat_srcs}) != 1:
            raise ValueError("the maps in feat_srcs must share shape, dtype and device")
        feat_srcs = torch.stack(list(feat_srcs))
    if not isinstance(feat_srcs, torch.Tensor) or feat_srcs.dim() != 5:
        raise ValueError("feat_srcs must be a [S,N,C,H,W] tensor or a sequence of [N,C,H,W] tensors")
    S = feat_srcs.shape[0]
    if S < 1:
        raise ValueError("feat_srcs has no source view")
    feat_src = feat_srcs.flatten(0, 1)                          # [S·N,C,H,W]: pair p = s·N + n
    if out is not None:
        if not isinstance(out, torch.Tensor) or out.dim() != 5 or out.shape != feat_srcs.shape:
            raise ValueError("out must be a [S,N,C,H,W] tensor")
        if out.shape[0] > 1 and out.shape[1] > 1 and out.stride(0) != out.shape[1] * out.stride(1):
            raise ValueError("out must be viewable as [S*N,C,H,W] (stride(0) == N * stride(1))")
    out4 = out.flatten(0, 1) if out is not None else None
    if isinstance(feat_ref, torch.Tensor) and (tuple(feat_srcs.shape[1:]) != tuple(feat_ref.shape) or feat_ref.device != feat_src.device):
        raise ValueError("feat_srcs must be [S,N,C,H,W] with [N,C,H,W] == feat_ref's shape, on feat_ref's device")
    if not isinstance(feat_ref, torch.Tensor) or feat_ref.dim() != 4:
        raise ValueError("feat_ref must be a 4-D tensor [N,C,H,W]")
    N, C, H, W = feat_ref.shape
    if sample_locs_in is None:
        if not isinstance(P_srcs, torch.Tensor) or tuple(P_srcs.shape) != (S, N, 3, 4):
            raise ValueError("P_srcs must be [S,N,3,4]")
        P_srcs = P_srcs.reshape(S * N, 3, 4)
    else:
        if tuple(sample_locs_in.shape) != (K, S, N, H, W, 2):
            raise ValueError("sample_locs_in must be [K,S,N,H,W,2]")
        sample_locs_in = sample_locs_in.reshape(K, S * N, H, W, 2)
    dcode = _check_feat_pair(feat_ref, feat_src, out4, out_dtype)
    if torch.is_grad_enabled() and (feat_ref.requires_grad or feat_src.requires_grad):
        raise RuntimeError("epipolar_fusion_multi is inference only (several sources have no backward); run it under "
                           "torch.no_grad(), or use epipolar_fusion (one source per call) for gradients")
    hp = None if head is None else _head_operands(lib, head, feat_ref, feat_src, out4, z_folded, z_residual, add_ref_residual)
    o, corr, attn, locs = _fusion(lib, dcode, S, feat_ref, feat_src, P_ref, P_srcs, K=K, downsample=downsample,
                                  img_scale=img_scale, softmax_scale=softmax_scale, correct_normalize=correct_normalize,
                                  align_corners=align_corners, z_folded=None if hp else z_folded, z_residual=z_residual and not hp,
                                  add_ref_residual=add_ref_residual and not hp, sample_locs_in=sample_locs_in, want_attn=want_attn,
                                  want_corr=want_corr, want_locs=want_locs, variant=variant, out=out4, state=state,
                                  out_dtype=out_dtype, head=hp)
    return (out if out is not None else o.unflatten(0, (S, N)), None if corr is None else corr.unflatten(0, (S, N)),
            None if attn is None else attn.unflatten(0, (S, N)), None if locs is None else locs.unflatten(1, (S, N)))


def view_source_table(sources, V):
    """A caller's source table as the C ABI takes it: [V,S] int32 on the host, every entry a view in [0, V) other than its
    row's own view (duplicates are allowed).  sources: a list of rows, a numpy array or a CPU integer tensor.  A CUDA tensor is
    refused: reading it back would synchronise the stream.  Build the table once per camera rig (`multiview.nearest_view_table`)."""
    if isinstance(sources, torch.Tensor):
        if sources.is_cuda:
            raise TypeError("sources must be on the host (a list, numpy array or CPU tensor): reading a CUDA table back would "
                            "synchronise the stream")
        if sources.dtype.is_floating_point or sources.dtype.is_complex or sources.dtype == torch.bool:
            raise TypeError("sources must hold integers (got %s)" % sources.dtype)
        sources = sources.numpy()
    t = np.asarray(sources)
    if t.ndim != 2 or t.shape[0] != V or t.shape[1] < 1:
        raise ValueError("sources must be a [V,S] table with V = %d rows and S >= 1 (got shape %s)" % (V, tuple(t.shape)))
    if t.dtype.kind not in "iu":
        raise TypeError("sources must hold integer view indices (got %s)" % t.dtype)
    if V * t.shape[1] > _lib.EPI_VIEW_SOURCES_MAX:
        raise ValueError("sources has %d entries; a call takes at most %d (V*S)" % (V * t.shape[1], _lib.EPI_VIEW_SOURCES_MAX))
    if (t < 0).any() or (t >= V).any():
        raise ValueError("sources entries must be views in [0, %d)" % V)
    own = np.nonzero(t == np.arange(V)[:, None])
    if own[0].size:
        raise ValueError("sources[%d] names view %d itself: a view is not fused with itself" % (own[0][0], own[0][0]))
    return np.ascontiguousarray(t, dtype=np.int32)


def epipolar_fusion_views(feats, P, *, K, downsample=4.0, img_scale=1.0, softmax_scale=0.125, correct_normalize=False,
                          align_corners=False, z_folded=None, z_residual=False, add_ref_residual=False, sample_locs_in=None,
                          want_attn=True, want_corr=True, want_locs=False, variant="auto", out=None,
                          state: Optional[FusionState] = None, sources=None, out_dtype=torch.float32, head=None):
    """Fuses each view of a frame with several other views in one call, staging each view's map once.

    sources=None: every view with every other view, the whole multi-view test of the reference (cfg.EPIPOLAR.MULTITEST,
    modeling/model.py:213-239), where each of the V views takes a turn as the reference; S = V−1 and view v's j-th source is
    u = j + (j >= v) (the other views in increasing order).
    sources=[V,S] table (list, numpy array or CPU integer tensor; see `view_source_table`): view v's j-th source is
    u = sources[v][j].  With the nearest camera per view (S = 1, `multiview.nearest_view_table`) this is the reference's
    standard test (modeling/model.py:240-247) from one backbone pass.

    feats: [V,N,C,H,W], or a sequence of V [N,C,H,W] maps (stacked), V >= 2; P: [V,N,3,4]; sample_locs_in: optional
    [K,V,S,N,H,W,2]; out: optional [V,S,N,C,H,W] of dtype out_dtype (float32, or bfloat16 / float16 as in `epipolar_fusion`).  Reference view v with its j-th source u gives, bit for bit, what
    `epipolar_fusion(feats[v], feats[u], P[v], P[u])` gives; every residual (add_ref_residual, also under z) adds feats[v][n].
    Returns (out [V,S,N,C,H,W], corr_pos [V,S,N,H,W,2] | None, attn [V,S,N,K,H,W] | None, sample_locs [K,V,S,N,H,W,2] | None);
    with a `head` (as in `epipolar_fusion`; its residual adds feats[v][n]) heat [V,S,N,J,H,W] in place of out.
    Inference only: inputs that require grad under grad mode raise RuntimeError.  `epipolar_fusion_views_backward` is its
    backward, and `Epipolar.forward_views_train` the differentiable form."""
    lib = _lib.load()
    if head is not None:
        _lib.require_heatmaps(lib)
    if isinstance(feats, (list, tuple)):
        if not all(isinstance(t, torch.Tensor) for t in feats):
            raise ValueError("feats must be a [V,N,C,H,W] tensor or a sequence of V [N,C,H,W] tensors")
        if len({(tuple(t.shape), t.dtype, t.device) for t in feats}) > 1:
            raise ValueError("the maps in feats must share shape, dtype and device")
        if len(feats) < 2:
            raise ValueError("feats needs at least two views (got %d)" % len(feats))
        feats = torch.stack(list(feats))
    if not isinstance(feats, torch.Tensor) or feats.dim() != 5:
        raise ValueError("feats must be a [V,N,C,H,W] tensor or a sequence of V [N,C,H,W] tensors")
    V, N, C, H, W = feats.shape
    if V < 2:
        raise ValueError("feats needs at least two views (got %d)" % V)
    table = None if sources is None else view_source_table(sources, V)
    if table is not None:
        _lib.require_view_sources(lib)
    S = V - 1 if table is None else table.shape[1]
    Sn = "V-1" if table is None else "S"                        # the sources dimension, as the messages name it
    feat = feats.flatten(0, 1)                                  # [V·N,C,H,W]: item v·N + n
    if out is not None:
        if not isinstance(out, torch.Tensor) or tuple(out.shape) != (V, S, N, C, H, W):
            raise ValueError("out must be a [V,%s,N,C,H,W] tensor" % Sn)
        try:
            out4 = out.view(V * S * N, C, H, W)
        except RuntimeError:
            raise ValueError("out must be viewable as [V*(%s)*N,C,H,W]" % Sn) from None
    else:
        out4 = None
    if sample_locs_in is None:
        if not isinstance(P, torch.Tensor) or tuple(P.shape) != (V, N, 3, 4):
            raise ValueError("P must be [V,N,3,4]")
        P = P.reshape(V * N, 3, 4)
    else:
        if tuple(sample_locs_in.shape) != (K, V, S, N, H, W, 2):
            raise ValueError("sample_locs_in must be [K,V,%s,N,H,W,2]" % Sn)
        sample_locs_in = sample_locs_in.reshape(K, V * S * N, H, W, 2)
    dcode = _check_feat_pair(feat, feat, out4, out_dtype)
    if torch.is_grad_enabled() and feat.requires_grad:
        raise RuntimeError("epipolar_fusion_views is inference only; run it under torch.no_grad(), or use "
                           "Epipolar.forward_views_train (backward: epipolar_fusion_views_backward) for gradients")
    hp = None if head is None else _head_operands(lib, head, feat, feat, out4, z_folded, z_residual, add_ref_residual)
    o, corr, attn, locs = _fusion(lib, dcode, 1, feat, None, P, None, K=K, downsample=downsample, img_scale=img_scale,
                                  softmax_scale=softmax_scale, correct_normalize=correct_normalize,
                                  align_corners=align_corners, z_folded=None if hp else z_folded, z_residual=z_residual and not hp,
                                  add_ref_residual=add_ref_residual and not hp, sample_locs_in=sample_locs_in, want_attn=want_attn,
                                  want_corr=want_corr, want_locs=want_locs, variant=variant, out=out4, state=state, views=V,
                                  table=table, out_dtype=out_dtype, head=hp)
    pairs = (V, S, N)
    return (out if out is not None else o.unflatten(0, pairs), None if corr is None else corr.unflatten(0, pairs),
            None if attn is None else attn.unflatten(0, pairs), None if locs is None else locs.unflatten(1, pairs))


def _fusion(lib, dcode, S, feat_ref, feat_src, P_ref, P_src, *, K, downsample, img_scale, softmax_scale, correct_normalize,
            align_corners, z_folded, z_residual, add_ref_residual, sample_locs_in, want_attn, want_corr, want_locs, variant, out,
            state, views=0, table=None, out_dtype=torch.float32, head=None):
    """The forward of `epipolar_fusion` (S = 1) and `epipolar_fusion_multi`: feat_ref [N,C,H,W], feat_src / out [S·N,C,H,W],
    P_src [S·N,3,4], sample_locs_in [K,S·N,H,W,2]; outputs have S·N items (pair p = s·N + n).
    views = V >= 2 (`epipolar_fusion_views`): feat_ref [V·N,C,H,W] and P_ref [V·N,3,4] hold the views, feat_src and P_src are
    None, and the outputs have V·S·N items (pair p = (v·S + j)·N + n), S = V−1, or the width of `table` ([V,S] int32 host
    array from `view_source_table`, which selects the source-table entry points).  out has dtype out_dtype.
    head = (A, B | None, b) from `_head_operands`: the heat-map call (epi_fusion_heatmaps_f32); `out` is then None, and the first
    result is heat [pairs,J,H,W] of dtype out_dtype."""
    NR, C, H, W = feat_ref.shape
    ocode = FEAT_DTYPES[out_dtype]
    N = NR // views if views else NR
    NP = views * (views - 1 if table is None else table.shape[1]) * N if views else S * N
    dev = feat_ref.device
    if sample_locs_in is None:
        if P_ref.device != dev or P_ref.dtype != torch.float32 or not P_ref.is_contiguous():
            P_ref = P_ref.to(device=dev, dtype=torch.float32).contiguous()
        if P_src is not None and (P_src.device != dev or P_src.dtype != torch.float32 or not P_src.is_contiguous()):
            P_src = P_src.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(P_ref.shape) != (NR, 3, 4) or (not views and tuple(P_src.shape) != (NP, 3, 4)):
            raise ValueError("P_ref/P_src must be [N,3,4]" if S == 1 else "P_ref must be [N,3,4] and P_srcs [S,N,3,4]")
    else:
        sample_locs_in = _aligned_locs(sample_locs_in.to(device=dev, dtype=torch.float32))
        if tuple(sample_locs_in.shape) != (K, NP, H, W, 2):
            raise ValueError("sample_locs_in must be [K,N,H,W,2]")
    if head is not None:
        out = torch.empty((NP, head[0].shape[0], H, W), device=dev, dtype=out_dtype)       # heat
    elif out is None and views:                                          # the layout of a single call's empty_like(feat_src)
        cl = feat_ref.dim() == 4 and feat_ref.is_contiguous(memory_format=torch.channels_last) and not feat_ref.is_contiguous()
        out = torch.empty((NP, C, H, W), device=dev, dtype=out_dtype,
                          memory_format=torch.channels_last if cl else torch.contiguous_format)
    elif out is None:
        out = torch.empty_like(feat_src, dtype=out_dtype)               # preserves NCHW / channels_last
    attn = torch.empty((NP, K, H, W), device=dev, dtype=torch.float32) if want_attn else None
    corr = torch.empty((NP, H, W, 2), device=dev, dtype=torch.float32) if want_corr else None
    locs = torch.empty((K, NP, H, W, 2), device=dev, dtype=torch.float32) if want_locs else None

    vcode = _lib.VARIANTS[variant] if isinstance(variant, str) else int(variant)
    # the plan (and so the workspace size) also depends on whether `out` and feat_src start on a 16-byte boundary
    src_key = (feat_src.stride(), feat_src.data_ptr() % 16 == 0) if feat_src is not None else (feat_ref.data_ptr() % 16 == 0,)
    tkey = None if table is None else (table.shape, table.tobytes())
    key = (dev, S, views, tkey, N, C, H, W, int(K), dcode, ocode, feat_ref.stride(), out.stride(), out.data_ptr() % 16 == 0, src_key,
           z_folded is not None, vcode,
           sample_locs_in is not None, float(downsample), float(img_scale), float(softmax_scale), bool(correct_normalize),
           bool(align_corners), bool(z_residual), bool(add_ref_residual), head is not None)
    if state is not None and state.key == key:
        p = state.params
    else:
        p = _lib.EpiFusionParams()
        p.ref_stride = _strides4(feat_ref); p.out_stride = _strides4(out)
        if feat_src is not None:
            p.src_stride = _strides4(feat_src)
        p.N, p.C, p.H, p.W, p.K = N, C, H, W, int(K)
        p.downsample = float(downsample); p.img_scale = float(img_scale)
        p.eps = _EPSILON; p.softmax_scale = float(softmax_scale)
        p.align_corners = int(bool(align_corners)); p.correct_normalize = int(bool(correct_normalize))
        p.z_residual = int(bool(z_residual)); p.add_ref_residual = int(bool(add_ref_residual))
        p.variant = vcode
        p.feat_dtype = dcode | _lib.EPI_OUT_DTYPE(ocode)
        p.n_src = S if S > 1 else 0
        p.n_views = views
    p.feat_ref = feat_ref.data_ptr(); p.feat_src = feat_src.data_ptr() if feat_src is not None else None
    p.P_ref = P_ref.data_ptr() if sample_locs_in is None else None
    p.P_src = P_src.data_ptr() if sample_locs_in is None and P_src is not None else None
    p.sample_locs_in = sample_locs_in.data_ptr() if sample_locs_in is not None else None
    p.out = out.data_ptr() if head is None else None
    p.attn = attn.data_ptr() if attn is not None else None
    p.corr_pos = corr.data_ptr() if corr is not None else None
    p.sample_locs_out = locs.data_ptr() if locs is not None else None
    if z_folded is not None:
        wf, bf = z_folded
        p.z_weight_folded = wf.data_ptr(); p.z_bias_folded = bf.data_ptr()
    if head is not None:                                           # the heat-map call: any form, with or without a table
        h = _lib.EpiHeadParams()
        A, B, b = head
        h.A = A.data_ptr(); h.B = B.data_ptr() if B is not None else None; h.b = b.data_ptr()
        h.heat = out.data_ptr(); h.heat_stride = _strides4(out); h.J = A.shape[0]
        targs = (ctypes.byref(h),) + ((None, 0) if table is None else
                                      (table.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), table.shape[1]))
        cache_bytes = lambda q: lib.epi_fusion_heatmaps_cache_bytes(q, *targs)
        workspace_bytes = lambda q: lib.epi_fusion_heatmaps_workspace_bytes(q, *targs)
        forward = lambda q, st: lib.epi_fusion_heatmaps_f32(q, *targs, st)
    elif table is None:
        cache_bytes, workspace_bytes = lib.epi_fusion_cache_bytes, lib.epi_fusion_workspace_bytes
        forward = lib.epi_fusion_forward_f32
    else:                                                          # the [V,S] host table goes with every call
        targs = (table.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), table.shape[1])
        cache_bytes = lambda q: lib.epi_fusion_view_sources_cache_bytes(q, *targs)
        workspace_bytes = lambda q: lib.epi_fusion_view_sources_workspace_bytes(q, *targs)
        forward = lambda q, st: lib.epi_fusion_view_sources_forward_f32(q, *targs, st)
    ws = None
    if state is not None and state.key == key:
        pass                                                       # workspace / cache pointers already in the block
    else:
        if state is not None:
            cbytes = cache_bytes(ctypes.byref(p))
            state.cache = torch.zeros(cbytes, device=dev, dtype=torch.uint8) if cbytes else None
            p.cache = state.cache.data_ptr() if cbytes else None
            p.cache_bytes = cbytes
        nbytes = workspace_bytes(ctypes.byref(p))
        if nbytes:
            ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)      # caching allocator: stream-ordered, 512-B aligned
            p.workspace = ws.data_ptr(); p.workspace_bytes = nbytes
        if state is not None:
            state.ws = ws; state.params = p; state.key = key
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(forward(ctypes.byref(p), ctypes.c_void_p(stream)), "epi_fusion_heatmaps_f32" if head is not None else
                   "epi_fusion_forward_f32" if table is None else "epi_fusion_view_sources_forward_f32")
    return out, corr, attn, locs


def epipolar_fusion_backward(feat_ref, feat_src, P_ref, P_src, attn, grad_out, *, K, downsample=4.0, img_scale=1.0,
                             softmax_scale=0.125, correct_normalize=False, align_corners=False, grad_attn=None,
                             sample_locs_in=None, grad_keys=True, grad_vals=True, need_ref=True, need_src=True,
                             deterministic=None):
    """Backward of `epipolar_fusion` without the z epilogue: returns (dL/dfeat_ref | None, dL/dfeat_src | None).
    Restates autograd through epipolar.py:188-247 (grid_sample x2, mul/sum, ==0 mask, softmax, weighted sum);
    grad_keys / grad_vals = 'other1' / 'other2' in cfg.EPIPOLAR.OTHER_GRAD (:141-153).
    The gradients have the maps' dtype (computed in float32, rounded once); grad_out is float32 like the forward's `out`.

    deterministic: None follows torch.are_deterministic_algorithms_enabled(); True / False force the path.  The deterministic
    path sums dL/dfeat_src in per-pair int64 fixed point, so identical inputs give identical bits whatever the rest of the batch
    and the layouts; it costs two more launches and more workspace (DESIGN.md §5).  A pair whose maps or gradients hold a NaN
    or inf gets an all-NaN dL/dfeat_src there.  dL/dfeat_ref is order-fixed, and the same bits, on both paths."""
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    elif not isinstance(deterministic, bool):
        raise TypeError("deterministic must be None or a bool (got %s)" % type(deterministic).__name__)
    lib = _lib.load()
    dcode = _check_feat_pair(feat_ref, feat_src)
    N, C, H, W = feat_ref.shape
    dev = feat_ref.device
    grad_out = grad_out if grad_out.dtype == torch.float32 else grad_out.float()
    attn = attn.contiguous()
    g_ref = torch.empty_like(feat_ref) if need_ref else None
    g_src = torch.empty_like(feat_src) if need_src else None
    if not need_ref and not need_src:
        return None, None
    p = _lib.EpiFusionBwdParams()
    p.feat_ref = feat_ref.data_ptr(); p.ref_stride = _strides4(feat_ref)
    p.feat_src = feat_src.data_ptr(); p.src_stride = _strides4(feat_src)
    if sample_locs_in is None:
        P_ref = P_ref.to(device=dev, dtype=torch.float32).contiguous(); P_src = P_src.to(device=dev, dtype=torch.float32).contiguous()
        p.P_ref = P_ref.data_ptr(); p.P_src = P_src.data_ptr()
    else:
        sample_locs_in = _aligned_locs(sample_locs_in.to(device=dev, dtype=torch.float32))
        p.sample_locs_in = sample_locs_in.data_ptr()
    p.attn = attn.data_ptr()
    p.grad_out = grad_out.data_ptr(); p.gout_stride = _strides4(grad_out)
    if grad_attn is not None:
        grad_attn = grad_attn.to(dtype=torch.float32).contiguous()
        p.grad_attn = grad_attn.data_ptr()
    if g_ref is not None:
        p.grad_ref = g_ref.data_ptr(); p.gref_stride = _strides4(g_ref)
    if g_src is not None:
        p.grad_src = g_src.data_ptr(); p.gsrc_stride = _strides4(g_src)
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, int(K)
    p.downsample = float(downsample); p.img_scale = float(img_scale); p.eps = _EPSILON; p.softmax_scale = float(softmax_scale)
    p.align_corners = int(bool(align_corners)); p.correct_normalize = int(bool(correct_normalize))
    p.grad_keys = int(bool(grad_keys)); p.grad_vals = int(bool(grad_vals))
    p.feat_dtype = dcode
    p.deterministic = int(deterministic)
    nbytes = lib.epi_fusion_backward_workspace_bytes(ctypes.byref(p))
    ws = torch.empty(max(nbytes, 1), device=dev, dtype=torch.uint8)
    p.workspace = ws.data_ptr(); p.workspace_bytes = nbytes
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.epi_fusion_backward_f32(ctypes.byref(p), ctypes.c_void_p(stream)), "epi_fusion_backward_f32")
    return g_ref, g_src


def epipolar_fusion_views_backward(feats, P, attn, grad_out, *, K, downsample=4.0, img_scale=1.0, softmax_scale=0.125,
                                   correct_normalize=False, align_corners=False, sources=None, grad_attn=None, sample_locs_in=None,
                                   grad_keys=True, grad_vals=True, deterministic=None):
    """Backward of `epipolar_fusion_views` without the z epilogue: dL/dfeats [V,N,C,H,W] in the maps' dtype (float32 sums,
    rounded once).  Each view item gets the dL/dfeat_ref terms of the pairs it is the query of and, as grad_keys / grad_vals
    ('other1' / 'other2' in cfg.EPIPOLAR.OTHER_GRAD) select, the dL/dfeat_src terms of the pairs that name it as their source;
    every term is what `epipolar_fusion_backward` computes for that pair.  A view that is nobody's source gets query terms only.

    feats: [V,N,C,H,W] (or V [N,C,H,W] maps); P: [V,N,3,4] (unused with sample_locs_in); attn, grad_attn: [V,S,N,K,H,W];
    grad_out: [V,S,N,C,H,W]; sample_locs_in: optional [K,V,S,N,H,W,2], the locations the forward sampled; sources: None (every
    other view) or a [V,S] host table, as in `epipolar_fusion_views`.  Each view map is staged once.
    deterministic: None follows torch.are_deterministic_algorithms_enabled(); True sums the source terms in per-item int64 fixed
    point, whose scale depends on the item's own frame only, so the bits do not depend on the rest of the batch or the layouts.
    An item one of whose source pairs has a NaN or inf in its maps or gradients comes out all NaN on that path."""
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    elif not isinstance(deterministic, bool):
        raise TypeError("deterministic must be None or a bool (got %s)" % type(deterministic).__name__)
    lib = _lib.load()
    if isinstance(feats, (list, tuple)):
        if len({(tuple(t.shape), t.dtype, t.device) for t in feats if isinstance(t, torch.Tensor)}) != 1 or \
                not all(isinstance(t, torch.Tensor) for t in feats):
            raise ValueError("the maps in feats must be tensors sharing shape, dtype and device")
        feats = torch.stack(list(feats))
    if not isinstance(feats, torch.Tensor) or feats.dim() != 5:
        raise ValueError("feats must be a [V,N,C,H,W] tensor or a sequence of V [N,C,H,W] tensors")
    V, N, C, H, W = feats.shape
    if V < 2:
        raise ValueError("feats needs at least two views (got %d)" % V)
    table = None if sources is None else view_source_table(sources, V)
    _lib.require_views_backward(lib)
    S = V - 1 if table is None else table.shape[1]
    Sn = "V-1" if table is None else "S"
    for name, t, shape in (("attn", attn, (V, S, N, K, H, W)), ("grad_out", grad_out, (V, S, N, C, H, W)),
                           ("grad_attn", grad_attn, (V, S, N, K, H, W))):
        if t is not None and (not isinstance(t, torch.Tensor) or tuple(t.shape) != shape):
            raise ValueError("%s must be a [V,%s,N,%s,H,W] tensor" % (name, Sn, "K" if name != "grad_out" else "C"))
    feat = feats.flatten(0, 1)                                  # [V·N,C,H,W]: item v·N + n
    dcode = _check_feat_pair(feat, feat)
    dev = feat.device
    NP = V * S * N
    grad_out = grad_out.reshape(NP, C, H, W)
    grad_out = grad_out if grad_out.dtype == torch.float32 else grad_out.float()
    attn = attn.reshape(NP, K, H, W).to(dtype=torch.float32).contiguous()
    g = torch.empty_like(feat)
    p = _lib.EpiFusionBwdParams()
    p.feat_ref = feat.data_ptr(); p.ref_stride = _strides4(feat)
    if sample_locs_in is None:
        if not isinstance(P, torch.Tensor) or tuple(P.shape) != (V, N, 3, 4):
            raise ValueError("P must be [V,N,3,4]")
        P = P.reshape(V * N, 3, 4).to(device=dev, dtype=torch.float32).contiguous()
        p.P_ref = P.data_ptr()
    else:
        if tuple(sample_locs_in.shape) != (K, V, S, N, H, W, 2):
            raise ValueError("sample_locs_in must be [K,V,%s,N,H,W,2]" % Sn)
        sample_locs_in = _aligned_locs(sample_locs_in.reshape(K, NP, H, W, 2).to(device=dev, dtype=torch.float32))
        p.sample_locs_in = sample_locs_in.data_ptr()
    p.attn = attn.data_ptr()
    p.grad_out = grad_out.data_ptr(); p.gout_stride = _strides4(grad_out)
    if grad_attn is not None:
        grad_attn = grad_attn.reshape(NP, K, H, W).to(dtype=torch.float32).contiguous()
        p.grad_attn = grad_attn.data_ptr()
    p.grad_ref = g.data_ptr(); p.gref_stride = _strides4(g)
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, int(K)
    p.downsample = float(downsample); p.img_scale = float(img_scale); p.eps = _EPSILON; p.softmax_scale = float(softmax_scale)
    p.align_corners = int(bool(align_corners)); p.correct_normalize = int(bool(correct_normalize))
    p.grad_keys = int(bool(grad_keys)); p.grad_vals = int(bool(grad_vals))
    p.feat_dtype = dcode
    p.deterministic = int(deterministic)
    targs = (V, None if table is None else table.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 0 if table is None else S)
    nbytes = lib.epi_fusion_views_backward_workspace_bytes(ctypes.byref(p), *targs)
    ws = torch.empty(max(nbytes, 1), device=dev, dtype=torch.uint8)
    p.workspace = ws.data_ptr(); p.workspace_bytes = nbytes
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.epi_fusion_views_backward_f32(ctypes.byref(p), *targs, ctypes.c_void_p(stream)), "epi_fusion_views_backward_f32")
    return g.unflatten(0, (V, N))


class _FusionFn(torch.autograd.Function):
    """The fused attention under autograd (no z epilogue: conv/BN stay in PyTorch when gradients are needed).
    The gradients of bfloat16 / float16 maps come back in their dtype; `out` has opts["fwd"]["out_dtype"] (float32 by
    default), and its gradient is upcast to float32 for the backward kernels.
    The backward samples at the locations the forward emitted rather than re-deriving them from the cameras: the forward
    kernels round the line geometry differently, and with ill-conditioned cameras a recomputation moves samples by
    thousandths of a feature pixel, enough to put the gradients ~1e-3 (relative) off the function the forward computed."""

    @staticmethod
    def forward(ctx, feat_ref, feat_src, P_ref, P_src, opts):
        with torch.no_grad():
            out, corr, attn, locs = epipolar_fusion(feat_ref, feat_src, P_ref, P_src, want_attn=True,
                                                    **dict(opts["fwd"], want_locs=True))
        ctx.save_for_backward(feat_ref, feat_src, P_ref, P_src, attn, locs)
        ctx.opts = opts
        if not opts["fwd"].get("want_locs", False):
            locs = None
        nd = [t for t in (corr, locs) if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return out, corr, attn, locs

    @staticmethod
    def backward(ctx, g_out, g_corr, g_attn, g_locs):
        feat_ref, feat_src, P_ref, P_src, attn, locs = ctx.saved_tensors
        o = ctx.opts
        if g_out is None:
            g_out = torch.zeros_like(feat_ref, dtype=torch.float32)
        need_ref, need_src = ctx.needs_input_grad[0], ctx.needs_input_grad[1] and (o["grad_keys"] or o["grad_vals"])
        f = o["fwd"]
        g_ref, g_src = epipolar_fusion_backward(
            feat_ref, feat_src, P_ref, P_src, attn, g_out, K=f["K"], downsample=f["downsample"], img_scale=f["img_scale"],
            softmax_scale=f["softmax_scale"], correct_normalize=f["correct_normalize"], align_corners=f["align_corners"],
            grad_attn=g_attn, sample_locs_in=locs, grad_keys=o["grad_keys"], grad_vals=o["grad_vals"], need_ref=need_ref,
            need_src=need_src, deterministic=None)          # read torch's flag now, as PyTorch's own ops do in their backward
        if ctx.needs_input_grad[1] and g_src is None:
            g_src = torch.zeros_like(feat_src)
        return g_ref, g_src, None, None, None


class _ViewsFusionFn(torch.autograd.Function):
    """The views form under autograd (no z epilogue), for the reason and in the way of `_FusionFn`: the forward saves the
    attention and the locations it sampled, and the backward (`epipolar_fusion_views_backward`) samples there.  feats
    [V,N,C,H,W] gets one gradient per view item, summed over the pairs it is the query or the source of."""

    @staticmethod
    def forward(ctx, feats, P, sources, opts):
        with torch.no_grad():
            out, corr, attn, locs = epipolar_fusion_views(feats, P, want_attn=True, sources=sources,
                                                          **dict(opts["fwd"], want_locs=True))
        ctx.save_for_backward(feats, attn, locs)
        ctx.opts, ctx.sources = opts, sources
        if not opts["fwd"].get("want_locs", False):
            locs = None
        nd = [t for t in (corr, locs) if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return out, corr, attn, locs

    @staticmethod
    def backward(ctx, g_out, g_corr, g_attn, g_locs):
        feats, attn, locs = ctx.saved_tensors
        o = ctx.opts
        f = o["fwd"]
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        if g_out is None:
            g_out = torch.zeros(attn.shape[:3] + feats.shape[2:], device=feats.device, dtype=torch.float32)
        g = epipolar_fusion_views_backward(
            feats, None, attn, g_out, K=f["K"], downsample=f["downsample"], img_scale=f["img_scale"],
            softmax_scale=f["softmax_scale"], correct_normalize=f["correct_normalize"], align_corners=f["align_corners"],
            sources=ctx.sources, grad_attn=g_attn, sample_locs_in=locs, grad_keys=o["grad_keys"], grad_vals=o["grad_vals"],
            deterministic=None)          # read torch's flag now, as PyTorch's own ops do in their backward
        return g, None, None, None


def fold_z_bn(z: nn.Conv2d, bn: nn.BatchNorm2d):
    """(Wf, bf) such that BN_eval(z(x)) == Wf·x + bf, computed on the device (no host sync), always float32.  Parameters of a
    module cast to bfloat16 / float16 (or held in any other layout) are read as their exact contiguous float32 upcast."""
    lib = _lib.load()
    C = z.out_channels
    dev = z.weight.device
    wf = torch.empty((C, z.in_channels), device=dev, dtype=torch.float32)
    bf = torch.empty((C,), device=dev, dtype=torch.float32)
    f32 = lambda t: None if t is None else t.detach().to(dtype=torch.float32).contiguous()      # no copy when already so
    zw, zb, g, b, mean, var = map(f32, (z.weight, z.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var))
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.epi_fold_z_bn_f32(zw.data_ptr(), zb.data_ptr() if zb is not None else None, g.data_ptr(), b.data_ptr(),
                                         mean.data_ptr(), var.data_ptr(), float(bn.eps), C,
                                         wf.data_ptr(), bf.data_ptr(), ctypes.c_void_p(stream)), "epi_fold_z_bn_f32")
    return wf, bf


def head_weights(head):
    """(weight [J,C], bias [J] | None) of a pose head: a 1x1 nn.Conv2d (stride 1, no padding, one group, like `final_layer`,
    resnet.py:421) or a (weight [J,C] or [J,C,1,1], bias [J] | None) pair.  Anything else raises ValueError."""
    if isinstance(head, nn.Conv2d):
        if (head.kernel_size != (1, 1) or head.stride != (1, 1) or head.dilation != (1, 1) or head.groups != 1 or
                tuple(head.padding) != (0, 0)):
            raise ValueError("the head must be a 1x1 nn.Conv2d with stride 1, no padding and one group (got %r)" % (head,))
        weight, bias = head.weight, head.bias
    elif isinstance(head, (tuple, list)) and len(head) == 2:
        weight, bias = head
    else:
        raise ValueError("head must be a 1x1 nn.Conv2d or a (weight, bias) pair (got %s)" % type(head).__name__)
    if not isinstance(weight, torch.Tensor) or not (weight.dim() == 2 or (weight.dim() == 4 and weight.shape[2:] == (1, 1))):
        raise ValueError("the head weight must be [J,C] or [J,C,1,1]")
    weight = weight.flatten(1)
    J = weight.shape[0]
    if not 1 <= J <= _lib.HEAD_MAX_JOINTS:
        raise ValueError("the head must have 1 to %d output channels (got %d)" % (_lib.HEAD_MAX_JOINTS, J))
    if bias is not None and (not isinstance(bias, torch.Tensor) or tuple(bias.shape) != (J,)):
        raise ValueError("the head bias must be None or [J]")
    return weight, bias


def fold_head(weight, bias=None, z_folded=None, z_residual=False):
    """(A [J,C], b [J]) of the heat-map epilogue, computed on the device (one launch, no host sync): A = Wh·(Wf + z_residual·I),
    b = Wh·bf + bh, each element summed in fp64 and rounded once to float32; without z_folded (a layer without z) A = Wh and
    b = bh.  weight [J,C] (or [J,C,1,1]) and bias [J] | None are read as their float32 values; z_folded = `fold_z_bn`'s (Wf, bf)."""
    lib = _lib.load()
    _lib.require_heatmaps(lib)
    weight, bias = head_weights((weight, bias))
    J, C = weight.shape
    dev = weight.device
    if not weight.is_cuda:
        raise RuntimeError("the head weight is on %s: the heat-map epilogue has no CPU implementation" % dev)
    f32 = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous()
    wh, bh = f32(weight), f32(bias)
    wf, bf = (None, None) if z_folded is None else map(f32, z_folded)
    if wf is not None and tuple(wf.shape) != (C, C):
        raise ValueError("z_folded's weight must be [C,C] with C = %d, the head's input channels" % C)
    A = torch.empty((J, C), device=dev, dtype=torch.float32)
    b = torch.empty((J,), device=dev, dtype=torch.float32)
    ptr = lambda t: None if t is None else t.data_ptr()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.epi_fold_head_f32(wh.data_ptr(), ptr(bh), ptr(wf), ptr(bf), int(bool(z_residual and wf is not None)), J, C,
                                         A.data_ptr(), b.data_ptr(), ctypes.c_void_p(stream)), "epi_fold_head_f32")
    return A, b


class _Folded(tuple):
    """(A, B, b) that `Epipolar._head_folded` folded and checked: the functional forms take it as their `head` as it stands."""


def _head_operands(lib, head, feat_ref, feat_src, out, z_folded, z_residual, add_ref_residual):
    """(A, B | None, b) of a functional heat-map call: z / BN folded into the head, B = the head weight with the caller's
    residual.  Refuses `out` and gradients (the heat-map forward has no backward)."""
    _lib.require_heatmaps(lib)
    if out is not None:
        raise ValueError("a call with a head returns heat-maps: out must be None (the fused feature is not stored)")
    if isinstance(head, _Folded):
        return tuple(head)
    weight, bias = head_weights(head)
    if weight.shape[1] != feat_ref.shape[1]:
        raise ValueError("the head takes %d channels, the maps have %d" % (weight.shape[1], feat_ref.shape[1]))
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (feat_ref, feat_src, weight, bias)):
        raise RuntimeError("the heat-map forward is inference only (it has no backward); run it under torch.no_grad()")
    A, b = fold_head(weight, bias, z_folded, z_residual)
    B = weight.detach().to(dtype=torch.float32).contiguous() if add_ref_residual else None
    return A, B, b


def sample_locs(P_ref, P_src, H, W, K, downsample=4.0, img_scale=1.0, correct_normalize=False):
    """Device grid2sample_locs (epipolar.py:323-418): [K,N,H,W,2] normalised (x,y)."""
    lib = _lib.load()
    P_ref = P_ref.to(dtype=torch.float32).contiguous(); P_src = P_src.to(dtype=torch.float32).contiguous()
    if not P_ref.is_cuda:
        raise RuntimeError("sample_locs needs CUDA tensors (no CPU implementation)")
    N = P_ref.shape[0]
    out = torch.empty((K, N, H, W, 2), device=P_ref.device, dtype=torch.float32)
    with torch.cuda.device(P_ref.device):
        stream = torch.cuda.current_stream(P_ref.device).cuda_stream
        _lib.check(lib.epi_sample_locs_f32(P_ref.data_ptr(), P_src.data_ptr(), out.data_ptr(), N, H, W, K, float(downsample),
                                           float(img_scale), _EPSILON, int(bool(correct_normalize)), ctypes.c_void_p(stream)),
                   "epi_sample_locs_f32")
    return out


class Epipolar(nn.Module):
    """Drop-in for the reference's `Epipolar` on the graded flag set
    (ATTENTION='avg', SIMILARITY='dot', SOFTMAX_ENABLED, optional 'z' + ZRESIDUAL).

    Extra keyword-only knobs (all default to the reference's behaviour):
      cfg               duck-typed config (defaults to the module-level one, like `from core import cfg`)
      align_corners     grid_sample semantics; False = what the reference does under torch>=1.3
      fuse_ref_residual also add feat1 inside the kernel (use `fused_other_feat` as the caller)
      variant           'auto' | 'warp' | 'tile' kernel selection

    Under torch.use_deterministic_algorithms(True) the training backward is bit-reproducible (see
    `epipolar_fusion_backward`); the flag is read when the backward runs.  The z conv and BatchNorm stay PyTorch's.

    The module follows the dtype it is cast to (`.to(torch.bfloat16)`, `.half()`, `.bfloat16()`): a 16-bit module returns
    its fused feature in that dtype, the float32 result rounded once (in eval the folded epilogue stores it directly; under
    autograd z, BatchNorm and the residual adds then run in the module's dtype).  A float32 module returns float32, with or
    without torch.autocast.
    """

    def __init__(self, debug=False, *, cfg=None, align_corners=False, fuse_ref_residual=False, variant="auto",
                 emit_attn=True, emit_corr=True):
        super().__init__()
        cfg = cfg if cfg is not None else get_global_cfg()
        self.cfg = cfg
        self.debug = debug
        self.downsample = cfg.BACKBONE.DOWNSAMPLE
        self.feat_h, self.feat_w = cfg.KEYPOINT.HEATMAP_SIZE
        self.sample_size = cfg.EPIPOLAR.SAMPLESIZE
        self.epsilon = _EPSILON
        self.align_corners = align_corners
        self.fuse_ref_residual = fuse_ref_residual
        self.variant = variant
        self.emit_attn = emit_attn
        self.emit_corr = emit_corr
        ep = cfg.EPIPOLAR
        unsupported = []
        if debug: unsupported.append("debug=True")
        if ep.ATTENTION != "avg": unsupported.append("ATTENTION=%r" % ep.ATTENTION)
        if ep.SIMILARITY != "dot": unsupported.append("SIMILARITY=%r" % ep.SIMILARITY)
        if not ep.SOFTMAX_ENABLED: unsupported.append("SOFTMAX_ENABLED=False")
        if ep.PRIOR or ep.PRIORMUL: unsupported.append("PRIOR")
        if ep.POOLING: unsupported.append("POOLING")
        if ep.BOTTLENECK != 1: unsupported.append("BOTTLENECK!=1")
        if ep.FIND_CORR != "feature": unsupported.append("FIND_CORR=%r" % ep.FIND_CORR)
        if ep.REPROJECT_LOSS_WEIGHT != 0: unsupported.append("REPROJECT_LOSS_WEIGHT")
        for name in ("theta", "phi", "g"):
            if name in ep.PARAMETERIZED: unsupported.append("PARAMETERIZED has %r" % name)
        if unsupported:
            raise NotImplementedError(
                "epipolar_transformers_b200 accelerates the graded flag set only (SURVEY.md 8a); "
                "not supported: " + ", ".join(unsupported))
        if "z" in ep.PARAMETERIZED:                                   # epipolar.py:63-65
            nf = cfg.KEYPOINT.NFEATS
            self.z = nn.Conv2d(nf // ep.BOTTLENECK, nf, kernel_size=1, stride=1, padding=0, bias=True)
            self.bn = ZeroInitBN(nf)
        self._fold_cache = None
        self._head_cache = None
        self._states = {}            # device -> FusionState (persistent workspace + camera-keyed cache)
        # carries the dtype the module is cast to, which `out` takes; no elements and not persistent, so the state_dict keys
        # stay the reference's
        self.register_buffer("_dtype_probe", torch.empty(0, dtype=torch.float32), persistent=False)

    @property
    def out_dtype(self):
        """dtype of the fused feature this module returns: the dtype it was cast to (float32, bfloat16 or float16)"""
        return self._dtype_probe.dtype

    # -- eval-mode folding of z + BN, cached on parameter versions -------------------------------
    def _folded(self):
        if torch.cuda.is_current_stream_capturing():
            # A CUDA graph folds inside itself (one launch per replay, reading the parameters in place): it then holds no
            # pointer to the cache below, which an eager call frees when a parameter changes, and no wait on an event recorded
            # outside the capture (which CUDA refuses), and its replays follow in-place parameter updates as eager calls do.
            return fold_z_bn(self.z, self.bn)
        ts = (self.z.weight, self.z.bias, self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var)
        key = tuple((t.data_ptr(), t._version) for t in ts if t is not None)
        dev = self.z.weight.device
        cur = torch.cuda.current_stream(dev)
        if self._fold_cache is None or self._fold_cache[0] != key:
            folded = fold_z_bn(self.z, self.bn)
            ev = torch.cuda.Event()
            ev.record(cur)
            self._fold_cache = (key, folded, ev, {cur.cuda_stream})
        _, folded, ev, seen = self._fold_cache
        if cur.cuda_stream not in seen:          # a consumer on another stream must not read the fold before it is written
            cur.wait_event(ev)
            seen.add(cur.cuda_stream)
        return folded

    # -- eval-mode folding of z + BN + the pose head into the heat-map epilogue, cached like _folded ---------------
    def _head_folded(self, head, feat):
        """(A, B, b) of the heat-map call for `head` (1x1 nn.Conv2d or (weight, bias)): z / BN (eval) folded into the head, and
        B = the head weight, which adds the caller's residual `ret + feat` (resnet.py:388).  Refuses gradients, and training
        mode with z."""
        lib = _lib.load()
        _lib.require_heatmaps(lib)
        weight, bias = head_weights(head)
        has_z = "z" in self.cfg.EPIPOLAR.PARAMETERIZED
        if has_z and self.training:
            raise RuntimeError("the heat-map forward folds the z projection's BatchNorm with its running statistics: call "
                               "module.eval() first")
        params = [weight, bias] + ([self.z.weight, self.z.bias, self.bn.weight, self.bn.bias] if has_z else [])
        if torch.is_grad_enabled() and (feat.requires_grad or any(t is not None and t.requires_grad for t in params)):
            raise RuntimeError("the heat-map forward is inference only (it has no backward); run it under torch.no_grad()")
        if weight.shape[1] != feat.shape[-3]:
            raise ValueError("the head takes %d channels, the maps have %d" % (weight.shape[1], feat.shape[-3]))
        zres = bool(self.cfg.EPIPOLAR.ZRESIDUAL) and has_z

        def fold():
            A, b = fold_head(weight, bias, self._folded() if has_z else None, zres)
            return A, weight.detach().to(dtype=torch.float32).contiguous(), b

        if torch.cuda.is_current_stream_capturing():
            return fold()                        # inside the graph, for the reason _folded gives
        ts = [weight, bias] + ([self.z.weight, self.z.bias, self.bn.weight, self.bn.bias, self.bn.running_mean,
                                self.bn.running_var] if has_z else [])
        key = (zres,) + tuple((t.data_ptr(), t._version) for t in ts if t is not None)
        cur = torch.cuda.current_stream(weight.device)
        if self._head_cache is None or self._head_cache[0] != key:
            folded = fold()
            ev = torch.cuda.Event()
            ev.record(cur)
            self._head_cache = (key, folded, ev, {cur.cuda_stream})
        _, folded, ev, seen = self._head_cache
        if cur.cuda_stream not in seen:          # a consumer on another stream must not read the fold before it is written
            cur.wait_event(ev)
            seen.add(cur.cuda_stream)
        return folded

    def _state_for(self, t, slot="single"):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            return None                                  # epipolar_fusion raises the proper error for CPU tensors
        return self._states.setdefault((t.device, torch.cuda.current_stream(t.device).cuda_stream, slot), FusionState())

    def forward(self, feat1, feat2, P1, P2, depth=None, camera=None, other_camera=None, ref1=None, ref2=None):
        """feat1/feat2: N x C x H x W; P1/P2: N x 3 x 4 (epipolar.py:82-89).
        Returns (finalout, corr_pos [N,H,W,2], depth=attention [N,K,H,W], sample_locs|None) (:262-269)."""
        if depth is not None:
            raise NotImplementedError("depth pass-through (epipolar.py:215-216) is not on the accelerated path")
        cfg = self.cfg
        ep = cfg.EPIPOLAR
        needs_grad = torch.is_grad_enabled() and (feat1.requires_grad or feat2.requires_grad)
        has_z = "z" in ep.PARAMETERIZED
        fold = has_z and not self.training and not needs_grad
        want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
        if needs_grad:
            # training: the fused attention runs under autograd (CUDA backward kernel); z conv + BN stay in PyTorch
            opts = dict(fwd=dict(K=self.sample_size, downsample=self.downsample,
                                 img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
                                 softmax_scale=ep.SOFTMAXSCALE, correct_normalize=ep.USE_CORRECT_NORMALIZE,
                                 align_corners=self.align_corners, want_corr=self.emit_corr, want_locs=want_locs,
                                 variant=self.variant, out_dtype=self.out_dtype),
                        grad_keys="other1" in ep.OTHER_GRAD, grad_vals="other2" in ep.OTHER_GRAD)
            out, corr, attn, locs = _FusionFn.apply(feat1, feat2, P1, P2, opts)
            if not self.emit_attn:
                attn = None
        else:
            out, corr, attn, locs = epipolar_fusion(
                feat1, feat2, P1, P2, K=self.sample_size, downsample=self.downsample,
                img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
                softmax_scale=ep.SOFTMAXSCALE, correct_normalize=ep.USE_CORRECT_NORMALIZE,
                align_corners=self.align_corners, z_folded=self._folded() if fold else None,
                z_residual=bool(ep.ZRESIDUAL) if fold else False,
                add_ref_residual=self.fuse_ref_residual and (fold or not has_z),
                want_attn=self.emit_attn, want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant,
                state=self._state_for(feat1), out_dtype=self.out_dtype)
        if has_z and not fold:
            # training-mode BN needs batch statistics (+ autograd to z/bn): keep conv/BN in PyTorch
            finalout = self.bn(self.z(out))
            if ep.ZRESIDUAL:
                finalout = finalout + out
            if self.fuse_ref_residual:
                finalout = finalout + feat1
        elif needs_grad and self.fuse_ref_residual:
            finalout = out + feat1
        else:
            finalout = out
        return finalout, corr, attn, (locs.transpose(0, 1) if want_locs else None)

    def forward_heatmaps(self, feat1, feat2, P1, P2, head):
        """The eval step of the pose network from this layer on, `head(fused_other_feat(feat1, feat2, P1, P2, self)[0])`
        (resnet.py:385-388,421), with the 1x1 head as the fused forward's epilogue: the fused feature is never stored.
        head: the 1x1 nn.Conv2d `final_layer` (or a (weight [J,C], bias [J]) pair), 1 <= J <= 64.  Returns (heat [N,J,H,W] in the
        module's dtype, corr_pos, attention, sample_locs) as `forward` returns them (bit for bit).  z / BN and the head are
        folded once per parameter version (`fold_head`).  Inference only: gradients and training mode with z raise
        RuntimeError."""
        cfg = self.cfg
        ep = cfg.EPIPOLAR
        hp = self._head_folded(head, feat1)
        want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
        heat, corr, attn, locs = epipolar_fusion(
            feat1, feat2, P1, P2, K=self.sample_size, downsample=self.downsample,
            img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE, softmax_scale=ep.SOFTMAXSCALE,
            correct_normalize=ep.USE_CORRECT_NORMALIZE, align_corners=self.align_corners, want_attn=self.emit_attn,
            want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant, state=self._state_for(feat1, "single-heat"),
            out_dtype=self.out_dtype, head=_Folded(hp))
        return heat, corr, attn, (locs.transpose(0, 1) if want_locs else None)

    def forward_multi(self, feat1, feats2, P1, P2s, head=None):
        """`forward` of one reference batch against S source views in one fused call (the MULTITEST path,
        modeling/model.py:213-239).  feat1 [N,C,H,W], feats2 [S,N,C,H,W] or a sequence of S [N,C,H,W] maps, P1 [N,3,4],
        P2s [S,N,3,4].  Returns what S calls of `forward` return, stacked over the sources:
        (finalout [S,N,C,H,W], corr_pos [S,N,H,W,2] | None, attention [S,N,K,H,W] | None, sample_locs [S,N,K,H,W,2] | None).
        Inference only.  With the z projection the module must be in eval mode: training-mode BatchNorm would take its
        batch statistics over all S·N items, which S separate calls do not.
        head: as in `forward_heatmaps`; then heat [S,N,J,H,W] = head(finalout + feat1) in place of finalout."""
        cfg = self.cfg
        ep = cfg.EPIPOLAR
        has_z = "z" in ep.PARAMETERIZED
        if head is not None:
            hp = self._head_folded(head, feat1)
            want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
            heat, corr, attn, locs = epipolar_fusion_multi(
                feat1, feats2, P1, P2s, K=self.sample_size, downsample=self.downsample,
                img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE, softmax_scale=ep.SOFTMAXSCALE,
                correct_normalize=ep.USE_CORRECT_NORMALIZE, align_corners=self.align_corners, want_attn=self.emit_attn,
                want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant, state=self._state_for(feat1, "multi-heat"),
                out_dtype=self.out_dtype, head=_Folded(hp))
            return heat, corr, attn, (locs.permute(1, 2, 0, 3, 4, 5) if want_locs else None)
        if has_z and self.training:
            raise RuntimeError("Epipolar.forward_multi with the z projection needs eval mode: training-mode BatchNorm statistics "
                               "over S*N items differ from S separate forward calls")
        want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
        out, corr, attn, locs = epipolar_fusion_multi(
            feat1, feats2, P1, P2s, K=self.sample_size, downsample=self.downsample,
            img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
            softmax_scale=ep.SOFTMAXSCALE, correct_normalize=ep.USE_CORRECT_NORMALIZE,
            align_corners=self.align_corners, z_folded=self._folded() if has_z else None,
            z_residual=bool(ep.ZRESIDUAL) if has_z else False, add_ref_residual=self.fuse_ref_residual,
            want_attn=self.emit_attn, want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant,
            state=self._state_for(feat1, "multi"), out_dtype=self.out_dtype)
        return out, corr, attn, (locs.permute(1, 2, 0, 3, 4, 5) if want_locs else None)

    def forward_views(self, feats, P, sources=None, head=None):
        """`forward` of every view of a frame against several other views in one fused call.  feats [V,N,C,H,W] or a
        sequence of V [N,C,H,W] maps, P [V,N,3,4].  sources=None: every other view (the whole MULTITEST path,
        modeling/model.py:213-239), S = V−1 and u = j + (j >= v); a [V,S] host table (see `epipolar_fusion_views`): u =
        sources[v][j].  Returns what `forward(feats[v], feats[u], P[v], P[u])` returns for reference view v and its j-th source
        u, stacked as (finalout [V,S,N,C,H,W], corr_pos [V,S,N,H,W,2] | None, attention [V,S,N,K,H,W] | None,
        sample_locs [V,S,N,K,H,W,2] | None).  Inference only.  With the z projection the module must be in eval mode, for the
        reason `forward_multi` gives.
        head: as in `forward_heatmaps`; then heat [V,S,N,J,H,W] = head(finalout + feats[v]) in place of finalout."""
        cfg = self.cfg
        ep = cfg.EPIPOLAR
        has_z = "z" in ep.PARAMETERIZED
        if head is not None:
            first = feats[0] if isinstance(feats, (list, tuple)) and feats else feats
            hp = self._head_folded(head, first)
            want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
            heat, corr, attn, locs = epipolar_fusion_views(
                feats, P, K=self.sample_size, downsample=self.downsample,
                img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE, softmax_scale=ep.SOFTMAXSCALE,
                correct_normalize=ep.USE_CORRECT_NORMALIZE, align_corners=self.align_corners, want_attn=self.emit_attn,
                want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant, state=self._state_for(first, "views-heat"),
                sources=sources, out_dtype=self.out_dtype, head=_Folded(hp))
            return heat, corr, attn, (locs.permute(1, 2, 3, 0, 4, 5, 6) if want_locs else None)
        if has_z and self.training:
            raise RuntimeError("Epipolar.forward_views with the z projection needs eval mode: training-mode BatchNorm statistics "
                               "over V*(V-1)*N items differ from separate forward calls")
        want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
        first = feats[0] if isinstance(feats, (list, tuple)) and feats else feats
        out, corr, attn, locs = epipolar_fusion_views(
            feats, P, K=self.sample_size, downsample=self.downsample,
            img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
            softmax_scale=ep.SOFTMAXSCALE, correct_normalize=ep.USE_CORRECT_NORMALIZE,
            align_corners=self.align_corners, z_folded=self._folded() if has_z else None,
            z_residual=bool(ep.ZRESIDUAL) if has_z else False, add_ref_residual=self.fuse_ref_residual,
            want_attn=self.emit_attn, want_corr=self.emit_corr, want_locs=want_locs, variant=self.variant,
            state=self._state_for(first, "views"), sources=sources, out_dtype=self.out_dtype)
        return out, corr, attn, (locs.permute(1, 2, 3, 0, 4, 5, 6) if want_locs else None)

    def forward_views_train(self, feats, P, sources=None):
        """The differentiable counterpart of `forward_views`, for training from one backbone pass: every view of a frame is
        fused with its sources (sources=None: every other view; a [V,S] host table, e.g. `multiview.nearest_view_table` with
        topk=1: the views it names), and gradients reach `feats` (honouring cfg.EPIPOLAR.OTHER_GRAD) and z / bn.
        feats [V,N,C,H,W] or V [N,C,H,W] maps, P [V,N,3,4].  Returns what `forward(feats[q], feats[u], P[q], P[u])` returns on
        the gathered batch of V·S·N pairs in pair order ((v·S + j)·N + n: query view v, source u = its j-th source), shaped
        (finalout [V,S,N,C,H,W], corr_pos [V,S,N,H,W,2] | None, attention [V,S,N,K,H,W] | None,
        sample_locs [V,S,N,K,H,W,2] | None).  The z conv and BatchNorm stay PyTorch's, over the V·S·N pair items, in training and
        eval mode; fuse_ref_residual adds feats[v] in PyTorch, as `forward` does under autograd."""
        cfg = self.cfg
        ep = cfg.EPIPOLAR
        has_z = "z" in ep.PARAMETERIZED
        want_locs = bool(cfg.VIS.EPIPOLAR_LINE)
        if isinstance(feats, (list, tuple)):
            feats = torch.stack(list(feats))
        opts = dict(fwd=dict(K=self.sample_size, downsample=self.downsample,
                             img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
                             softmax_scale=ep.SOFTMAXSCALE, correct_normalize=ep.USE_CORRECT_NORMALIZE,
                             align_corners=self.align_corners, want_corr=self.emit_corr, want_locs=want_locs,
                             variant=self.variant, out_dtype=self.out_dtype),
                    grad_keys="other1" in ep.OTHER_GRAD, grad_vals="other2" in ep.OTHER_GRAD)
        out, corr, attn, locs = _ViewsFusionFn.apply(feats, P, sources, opts)
        if not self.emit_attn:
            attn = None
        finalout = out
        if has_z:
            pairs = out.shape[:3]
            finalout = self.bn(self.z(out.flatten(0, 2))).unflatten(0, pairs)
            if ep.ZRESIDUAL:
                finalout = finalout + out
        if self.fuse_ref_residual:
            finalout = finalout + feats[:, None]             # the pair's query view feats[v], over its S sources
        return finalout, corr, attn, (locs.permute(1, 2, 3, 0, 4, 5, 6) if want_locs else None)


def fused_other_feat(feat, other_features, KRT, other_KRT, sampler: Epipolar, camera=None, other_camera=None):
    """Caller-side mirror of getOtherFeat (modeling/backbones/resnet.py:377-388):
    returns (ret + feat, corr_pos, depth, sample_locs).  With sampler.fuse_ref_residual the add
    already happened inside the kernel."""
    if other_features is None:
        return feat, None, None, None
    ret, corr_pos, depth, locs = sampler(feat, other_features, KRT, other_KRT, camera=camera, other_camera=other_camera)
    if not sampler.fuse_ref_residual:
        ret = ret + feat
    return ret, corr_pos, depth, locs


def _fused_tail(tail, fuse_head):
    """fuse_head=True needs `tail` to be the 1x1 head itself (an nn.Conv2d that `head_weights` accepts)."""
    if fuse_head:
        if not isinstance(tail, nn.Conv2d):
            raise ValueError("fuse_head=True needs tail to be the 1x1 nn.Conv2d head (got %s)" % type(tail).__name__)
        head_weights(tail)
    return fuse_head


def multitest(sampler: Epipolar, tail, feat, other_feats, KRT, other_KRTs, sigma, downsample, fuse_head=False):
    """The multi-view test of the reference (cfg.EPIPOLAR.MULTITEST, modeling/model.py:213-239) from the fusion layer on:
    every reference item is fused with each of the S other views, each fusion goes through the rest of the network and the
    peak finder, and every joint keeps the location of the source whose peak scores highest (torch.max over the sources, then
    gather).  Here the S fusions are one `Epipolar.forward_multi` call and the selection is one launch.

    feat [N,C,H,W] (the reference views' features at the merge point), other_feats [S,N,C,H,W] or S [N,C,H,W] maps, KRT
    [N,3,4], other_KRTs [S,N,3,4]; tail: everything after the merge point ([B,C,H,W] -> heat-maps [B,J,h,w]; `final_layer`
    for MERGE='late'); sigma = cfg.KEYPOINT.SIGMA, downsample as for find_tensor_peak_batch.
    Returns (locs [N,J,2], scores [N,J], source index [N,J]); the reference's final `squeeze()` is left to the caller.
    fuse_head=True: tail must be the 1x1 nn.Conv2d head (else ValueError), and runs as the fused forward's epilogue
    (`Epipolar.forward_multi(head=)`), so the fused feature is never stored."""
    if _fused_tail(tail, fuse_head):
        with torch.no_grad():
            heat, _, _, _ = sampler.forward_multi(feat, other_feats, KRT, other_KRTs, head=tail)
            return find_tensor_peak_best(heat, sigma, downsample)
    with torch.no_grad():
        ret, _, _, _ = sampler.forward_multi(feat, other_feats, KRT, other_KRTs)
        x = ret if sampler.fuse_ref_residual else ret + feat          # getOtherFeat's `ret + feat` (resnet.py:388), per source
        S, N = x.shape[0], x.shape[1]
        heat = tail(x.flatten(0, 1))
        return find_tensor_peak_best(heat.unflatten(0, (S, N)), sigma, downsample)


_device_tables = {}          # (device, shape, bytes) -> the [V,S] source table as an int64 device tensor


def _table_on(table, dev):
    """The source table on `dev`, copied once per (table, device): the per-step path makes no host-to-device copy."""
    key = (str(dev), table.shape, table.tobytes())
    t = _device_tables.get(key)
    if t is None:
        t = _device_tables[key] = torch.from_numpy(table.astype(np.int64)).to(dev)
    return t


def multitest_views(sampler: Epipolar, tail, feats, KRT, sigma, downsample, sources=None, fuse_head=False):
    """The reference's multi-view test (cfg.EPIPOLAR.MULTITEST, modeling/model.py:213-239) for every view of a frame at once:
    each view v is the reference in turn, is fused with each of its sources, each fusion goes through the rest of the
    network and the peak finder, and every joint keeps the location of the source whose peak scores highest.  All V·S
    fusions are one `Epipolar.forward_views` call and the selection is one launch of `find_tensor_peak_best`.

    feats [V,N,C,H,W] or V [N,C,H,W] maps (the views' features at the merge point), KRT [V,N,3,4]; tail, sigma and downsample
    as for `multitest`.  sources=None: every other view (S = V−1); a [V,S] host table (e.g. `multiview.nearest_view_table`
    with topk = S): the sources it names, a cheaper test over each view's S nearest cameras.  Returns per view
    (locs [V,N,J,2], scores [V,N,J], source view [V,N,J]): the source is the camera index u of the winning view, not its
    position j among the view's sources.
    fuse_head=True: tail must be the 1x1 nn.Conv2d head (else ValueError), and runs as the fused forward's epilogue
    (`Epipolar.forward_views(head=)`), so the V·S·N fused features are never stored."""
    fuse_head = _fused_tail(tail, fuse_head)
    with torch.no_grad():
        if isinstance(feats, (list, tuple)):
            feats = torch.stack(list(feats))
        if fuse_head:
            heat, _, _, _ = sampler.forward_views(feats, KRT, sources=sources, head=tail)
            V, S, N = heat.shape[0], heat.shape[1], heat.shape[2]
            heat = heat.flatten(0, 2)                                      # [V·S·N, J, h, w]
        else:
            ret, _, _, _ = sampler.forward_views(feats, KRT, sources=sources)
            V, S, N = ret.shape[0], ret.shape[1], ret.shape[2]
            x = ret if sampler.fuse_ref_residual else ret + feats[:, None]    # getOtherFeat's `ret + feat` of reference view v
            heat = tail(x.flatten(0, 2))                                       # [V·S·N, J, h, w]
        # [S, V·N, J, h, w]: source slot j of every (view, item)
        heat = heat.unflatten(0, (V, S, N)).transpose(0, 1).flatten(1, 2)
        locs, scores, j = find_tensor_peak_best(heat, sigma, downsample)
        j = j.unflatten(0, (V, N))
        if sources is None:
            v = torch.arange(V, device=j.device).view(V, 1, 1)
            return locs.unflatten(0, (V, N)), scores.unflatten(0, (V, N)), j + (j >= v).long()
        table = _table_on(view_source_table(sources, V), j.device)        # [V,S]
        return locs.unflatten(0, (V, N)), scores.unflatten(0, (V, N)), table.gather(1, j.flatten(1)).view_as(j)


def standard_views_test(sampler: Epipolar, tail, feats, KRT, sources, sigma, downsample, fuse_head=False):
    """The reference's standard (non-MULTITEST) test from one backbone pass: each view v is the reference once, fused with
    the one source view sources[v][0] (its nearest camera, data/datasets/multiview_h36m.py:231-238), and the fusion goes
    through getOtherFeat's residual (modeling/backbones/resnet.py:377-388), the rest of the network and the peak finder
    (resnet.py:423-430).  The reference runs the backbone a second time on the permuted views (modeling/model.py:240-247);
    here the other view's map is the same backbone output, so the V fusions are one `Epipolar.forward_views` call.

    sampler: the Epipolar layer; tail: everything after the merge point ([B,C,H,W] -> heat-maps [B,J,h,w]); feats
    [V,N,C,H,W] or V [N,C,H,W] maps (the views' features at the merge point); KRT [V,N,3,4]; sources: a [V,1] host table
    (`multiview.nearest_view_table(..., topk=1)`); sigma = cfg.KEYPOINT.SIGMA, downsample as for find_tensor_peak_batch.
    Returns per view (locs [V,N,J,2], scores [V,N,J], corr_pos [V,N,H,W,2] | None, attention [V,N,K,H,W] | None).
    fuse_head=True: tail must be the 1x1 nn.Conv2d head (else ValueError), and runs as the fused forward's epilogue
    (`Epipolar.forward_views(head=)`), so the fused features are never stored."""
    fuse_head = _fused_tail(tail, fuse_head)
    with torch.no_grad():
        if isinstance(feats, (list, tuple)):
            feats = torch.stack(list(feats))
        V, N = feats.shape[0], feats.shape[1]
        if view_source_table(sources, V).shape[1] != 1:
            raise ValueError("the standard test fuses each view with one source: sources must be [V,1]")
        if fuse_head:
            heat, corr, attn, _ = sampler.forward_views(feats, KRT, sources=sources, head=tail)
            heat = heat[:, 0].flatten(0, 1)
        else:
            ret, corr, attn, _ = sampler.forward_views(feats, KRT, sources=sources)
            x = ret[:, 0] if sampler.fuse_ref_residual else ret[:, 0] + feats     # getOtherFeat's `ret + feat`
            heat = tail(x.flatten(0, 1))
        locs, scores = find_tensor_peak_batch(heat, sigma, downsample)
        return (locs.unflatten(0, (V, N)), scores.unflatten(0, (V, N)), None if corr is None else corr[:, 0],
                None if attn is None else attn[:, 0])
