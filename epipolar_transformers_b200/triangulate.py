"""3-D joints from the views' 2-D joints on the GPU: the reference's KEYPOINT.TRIANGULATION = 'pymvg' mode.

The reference copies the locations, scores and cameras to the host and triangulates one frame at a time, one SVD per joint
(modeling/model.py, vision/triangulation.py's triangulate_pymvg, pymvg's find3d).  Here every (frame, joint) of a batch is one
thread of one launch (csrc/epi_triangulate.cu), with no host synchronisation, so the eval step can stay on the GPU and inside
a CUDA graph.  No CPU fallback.
"""
from __future__ import annotations

import ctypes
import math

import torch

from . import _lib


def triangulate_views(locs: torch.Tensor, scores: torch.Tensor, P: torch.Tensor, conf_thres: float = 0.05):
    """locs [V,N,J,2] (image px), scores [V,N,J], P [V,N,3,4] -> (X [N,J,3] float64, n_used [N,J] int32).

    The layout is that of `standard_views_test` / `multitest_views` (per view, per frame) and of `forward_views`' cameras.
    For each (frame n, joint j), as the reference's pymvg mode with zero distortion:
      1. the views: t = conf_thres; v is selected when scores[v,n,j] > t, compared in float32; while at most one view is
         selected and t >= -1, t drops by 0.05 (stepped in float64, as the reference's Python float);
      2. per selected view, in view order, the rows x·M[2] - M[0] and y·M[2] - M[1] of A, with M = P[v,n] in float64;
      3. X = w[:3] / w[3], w the right singular vector of A's smallest singular value.
    n_used is the number of views selected; X is NaN where it is below 2, or where a selected view's location or camera is
    not finite.  locs must already be in the cameras' pixels (the reference's IMAGE_RESIZE · PREDICT_RESIZE applied).
    locs and scores of another float dtype are read as float32.  P may be float32 (the layer's KRT) or float64; for pymvg's
    exact M pass K.double() @ RT.double().  One launch on the current stream; no host synchronisation."""
    lib = _lib.load()
    _lib.require_triangulate(lib)
    for name, t in (("locs", locs), ("scores", scores), ("P", P)):
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise ValueError("%s must be a floating-point tensor" % name)
    if locs.dim() != 4 or locs.shape[-1] != 2:
        raise ValueError("locs must be [V,N,J,2] (got %s)" % (tuple(locs.shape),))
    V, N, J = locs.shape[:3]
    if tuple(scores.shape) != (V, N, J):
        raise ValueError("scores must be [V,N,J] = %s (got %s)" % ((V, N, J), tuple(scores.shape)))
    if tuple(P.shape) != (V, N, 3, 4):
        raise ValueError("P must be [V,N,3,4] = %s (got %s)" % ((V, N, 3, 4), tuple(P.shape)))
    if not 2 <= V <= _lib.TRIANGULATE_MAX_VIEWS:
        raise ValueError("need 2 to %d views (got V = %d)" % (_lib.TRIANGULATE_MAX_VIEWS, V))
    if N < 1 or J < 1 or N * J > 2 ** 31 - 1:
        raise ValueError("need 1 <= N·J <= 2^31 - 1 (got N = %d, J = %d)" % (N, J))
    conf_thres = float(conf_thres)
    if not math.isfinite(conf_thres) or conf_thres > 1000.0:
        raise ValueError("conf_thres must be finite and at most 1000 (got %r)" % conf_thres)
    if not (locs.is_cuda and scores.is_cuda and P.is_cuda):
        raise RuntimeError("locs, scores and P are on %s, %s and %s: the CUDA triangulation has no CPU implementation"
                           % (locs.device, scores.device, P.device))
    if not locs.device == scores.device == P.device:
        raise ValueError("locs, scores and P must be on one device (got %s, %s and %s)" % (locs.device, scores.device, P.device))
    l = locs.detach().to(torch.float32).contiguous()
    s = scores.detach().to(torch.float32).contiguous()
    p = P.detach()
    p = (p if p.dtype == torch.float64 else p.to(torch.float32)).contiguous()
    dtype = _lib.EPI_DTYPE_F64 if p.dtype == torch.float64 else _lib.EPI_DTYPE_F32
    X = torch.empty((N, J, 3), device=l.device, dtype=torch.float64)
    n_used = torch.empty((N, J), device=l.device, dtype=torch.int32)
    with torch.cuda.device(l.device):
        stream = torch.cuda.current_stream(l.device).cuda_stream
        _lib.check(lib.epi_triangulate_dlt_f64(l.data_ptr(), s.data_ptr(), p.data_ptr(), dtype, conf_thres, V, N, J, X.data_ptr(),
                                               n_used.data_ptr(), ctypes.c_void_p(stream)), "epi_triangulate_dlt_f64")
    return X, n_used
