"""Host-side projective helpers with the reference's names and argument meaning
(/root/reference/vision/multiview.py).  The per-pixel versions used on the hot path live in
csrc/epi_common.cuh; these are the small per-camera utilities callers (datasets, visualisers,
the multi-GPU driver) use.  Unlike the reference, normalize/de_normalize take the flag
explicitly and never mutate their argument."""
from __future__ import annotations

import numpy as np
import torch


def camera_center(KRT, engine="numpy"):
    """C = -A^-1 t with A = KRT[..., :3] (multiview.py:8-23). numpy: ([3], invA); torch: ([N,4,1] homogeneous, invA)."""
    if engine == "numpy":
        invA = np.linalg.inv(KRT[:, :3])
        return -(invA @ KRT[:, 3]), invA
    if engine == "torch":
        invA = torch.inverse(KRT[..., :3])
        center = -torch.matmul(invA, KRT[..., 3, None])
        out = torch.ones([center.shape[0], 4, 1], dtype=KRT.dtype, device=center.device)
        out[..., :3, :] = center
        return out, invA
    raise ValueError(engine)


def pix2coord(x, downsample):
    """feature-pixel index -> image coordinate of its centre (multiview.py:154-157)."""
    return x * downsample + downsample / 2.0 - 0.5


def coord2pix(y, downsample):
    """inverse of pix2coord (multiview.py:159-163)."""
    return (y + 0.5 - downsample / 2.0) / downsample


def normalize(pts, H, W, correct=False):
    """feature px (x,y) -> grid_sample [-1,1] coordinates (multiview.py:25-37)."""
    out = pts.clone() if isinstance(pts, torch.Tensor) else np.array(pts, dtype=np.float64, copy=True)
    if correct:
        out[..., 0] = -1.0 + 2.0 * pts[..., 0] / (W - 1)
        out[..., 1] = -1.0 + 2.0 * pts[..., 1] / (H - 1)
    else:
        out[..., 0] = -1.0 + 2.0 * (pts[..., 0] + 0.5) / W
        out[..., 1] = -1.0 + 2.0 * (pts[..., 1] + 0.5) / H
    return out


def de_normalize(pts, H, W, correct=False):
    """inverse of normalize (multiview.py:39-57)."""
    out = pts.clone() if isinstance(pts, torch.Tensor) else np.array(pts, dtype=np.float64, copy=True)
    if correct:
        out[..., 0] = (pts[..., 0] + 1) * (W - 1) / 2.0
        out[..., 1] = (pts[..., 1] + 1) * (H - 1) / 2.0
    else:
        out[..., 0] = (pts[..., 0] + 1) * W / 2.0 - 0.5
        out[..., 1] = (pts[..., 1] + 1) * H / 2.0 - 0.5
    return out


def neighbor_cameras(centers, topk=1):
    """For each camera the indices of its `topk` nearest other cameras by centre distance
    (multiview.py:59-83 builds the same ranking per camera id)."""
    C = np.asarray(centers, dtype=np.float64)
    d = np.linalg.norm(C[:, None] - C[None], axis=-1)
    np.fill_diagonal(d, np.inf)
    return np.argsort(d, axis=1, kind="stable")[:, :topk]


def nearest_view_table(KRT_all, topk=1) -> np.ndarray:
    """The [V,topk] source table of `epipolar_fusion_views(..., sources=)`: for each view of a rig its `topk` nearest other
    cameras by centre distance, nearest first (`neighbor_cameras`; topk=1 is the pairing of the reference's standard test,
    data/datasets/multiview_h36m.py:231-238).  KRT_all: [V,3,4] (numpy or tensor, any device).  The cameras are constants of
    a rig, so compute the table once: reading a device tensor here synchronises."""
    K = KRT_all.detach().cpu().numpy() if isinstance(KRT_all, torch.Tensor) else np.asarray(KRT_all)
    K = K.astype(np.float64)
    if K.ndim != 3 or K.shape[1:] != (3, 4) or not 1 <= topk <= max(K.shape[0] - 1, 1):
        raise ValueError("need KRT_all [V,3,4] and 1 <= topk <= V-1 (got %s, topk=%d)" % (K.shape, topk))
    centers = np.stack([-np.linalg.solve(P[:, :3], P[:, 3]) for P in K])
    return neighbor_cameras(centers, topk=topk).astype(np.int32)
