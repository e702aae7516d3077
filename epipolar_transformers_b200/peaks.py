"""find_tensor_peak_batch on the GPU — the step right after the fusion layer's 1x1 head.

Mirrors /root/reference/modeling/backbones/basic_batch.py:17-63 (same name, arguments and return value for a
[J,H,W] heat-map) and adds the batched form the caller's Python loop (modeling/backbones/resnet.py:423-428) needs:
a [B,J,H,W] stack in one launch.  All arithmetic runs in libepipolar_b200.so (csrc/epi_peaks.cu); no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib


def _check_radius(radius):
    """The radius refusals of the C ABI, raised before any tensor work: not finite and > 0, or an R = int(radius + 0.5)
    (float32, as the kernel rounds it) outside 1 .. PEAKS_MAX_R, whose (2R+1)^2-sample window the kernel counts in int32."""
    if not (radius > 0) or not math.isfinite(radius):
        raise ValueError("The radius is not ok : %r" % (radius,))
    if radius >= _lib.PEAKS_MAX_R + 1 or int(np.float32(radius) + np.float32(0.5)) > _lib.PEAKS_MAX_R:
        raise ValueError("The radius is too large : %r (R = int(radius + 0.5) must be at most %d)" % (radius, _lib.PEAKS_MAX_R))


def _check_joints(B, J):
    if B * J > (2 ** 31 - 1) // 32:
        raise ValueError("B * J = %d is too large: one warp per joint, counted in int32" % (B * J))


def find_tensor_peak_batch(heatmap: torch.Tensor, radius, downsample, threshold: float = 0.000001, int_div: bool = False):
    """heatmap [J,H,W] -> (locs [J,2] (x, y), score [J]);  heatmap [B,J,H,W] -> ([B,J,2], [B,J]).

    int_div=False reproduces what the reference computes under current torch (`index / W` is a true division,
    basic_batch.py:26); int_div=True is the integer division of the torch < 1.4 the reference's README targets.

    Non-finite values follow the reference: a map holding a NaN has the first NaN as its score (torch.max), and the window
    keeps NaN through the threshold, so its location is NaN too.  bfloat16 and float16 maps are widened to float32 exactly
    and the peak is computed in float32, so they give the result of their float32 copy."""
    lib = _lib.load()
    if not isinstance(heatmap, torch.Tensor) or heatmap.dim() not in (3, 4):
        raise ValueError("The dimension of the heatmap is wrong : %s" % (tuple(heatmap.shape),))
    _check_radius(radius)
    if heatmap.shape[-2] <= 1 or heatmap.shape[-1] <= 1:
        raise ValueError("To avoid the normalization function divide zero")
    batched = heatmap.dim() == 4
    _check_joints(heatmap.shape[0] if batched else 1, heatmap.shape[-3])
    if not heatmap.is_cuda:
        raise RuntimeError("heatmap is on %s: the CUDA peak finder has no CPU implementation" % heatmap.device)
    h = heatmap if batched else heatmap.unsqueeze(0)
    h = h.detach().to(torch.float32).contiguous()
    B, J, H, W = h.shape
    locs = torch.empty((B, J, 2), device=h.device, dtype=torch.float32)
    score = torch.empty((B, J), device=h.device, dtype=torch.float32)
    with torch.cuda.device(h.device):
        stream = torch.cuda.current_stream(h.device).cuda_stream
        _lib.check(lib.epi_find_peaks_f32(h.data_ptr(), locs.data_ptr(), score.data_ptr(), B, J, H, W, float(radius),
                                          float(downsample), float(threshold), int(bool(int_div)), ctypes.c_void_p(stream)),
                   "epi_find_peaks_f32")
    return (locs, score) if batched else (locs[0], score[0])


def find_tensor_peak_best(heatmaps: torch.Tensor, radius, downsample, threshold: float = 0.000001, int_div: bool = False):
    """heatmaps [S,B,J,H,W] (S source views) -> (locs [B,J,2], scores [B,J], src_index [B,J] int64).

    The best-source selection of the reference's multi-view test (modeling/model.py:229-234): every source's peaks are
    `find_tensor_peak_batch` of its [B,J,H,W] stack, and each (b, j) keeps the peak of the source with the highest score,
    the first one on a tie, and the first source whose score is NaN if there is one (torch.max over sources, then gather).
    One launch for all sources; the radius and B·J limits are those of `find_tensor_peak_batch`."""
    lib = _lib.load()
    if not isinstance(heatmaps, torch.Tensor) or heatmaps.dim() != 5:
        raise ValueError("heatmaps must be [S,B,J,H,W] (got %s)" % (tuple(getattr(heatmaps, "shape", ())),))
    S, B, J, H, W = heatmaps.shape
    if min(S, B, J) < 1:
        raise ValueError("heatmaps has an empty dimension: %s" % (tuple(heatmaps.shape),))
    if H <= 1 or W <= 1:
        raise ValueError("To avoid the normalization function divide zero")
    _check_radius(radius)
    _check_joints(B, J)
    if not heatmaps.is_cuda:
        raise RuntimeError("heatmaps is on %s: the CUDA peak finder has no CPU implementation" % heatmaps.device)
    h = heatmaps.detach().to(torch.float32).contiguous()
    locs = torch.empty((B, J, 2), device=h.device, dtype=torch.float32)
    score = torch.empty((B, J), device=h.device, dtype=torch.float32)
    src = torch.empty((B, J), device=h.device, dtype=torch.int32)
    with torch.cuda.device(h.device):
        stream = torch.cuda.current_stream(h.device).cuda_stream
        _lib.check(lib.epi_find_peaks_best_f32(h.data_ptr(), locs.data_ptr(), score.data_ptr(), src.data_ptr(), S, B, J, H, W,
                                               float(radius), float(downsample), float(threshold), int(bool(int_div)),
                                               ctypes.c_void_p(stream)), "epi_find_peaks_best_f32")
    return locs, score, src.long()                       # int64 like the indices of torch.max
