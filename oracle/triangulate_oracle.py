"""TEST INFRASTRUCTURE — numpy restatement of the reference's KEYPOINT.TRIANGULATION = 'pymvg' mode, the oracle of
epi_triangulate_dlt_f64 (csrc/epi_triangulate.cu).  NOT product code.

Per (frame, joint), from the views' image-pixel locations, scores and 3x4 cameras M (fp64):
  1. views: t = conf_thres as a Python float; repeat { sel = {v : score[v] > t}; stop if t < -1; if |sel| <= 1, t -= 0.05
     (fp64, so the rounding accumulates) and repeat; else stop }.  The compare is float32 (numpy compares a float32 array
     with a Python float at float32), so float32(0.05) is not above 0.05, and a NaN score is never selected.
  2. A: per selected view, in increasing view order, the rows x·M[2] - M[0] and y·M[2] - M[1] (pymvg's find3d; with zero
     distortion its undistort is the identity).
  3. X = w[:3] / w[3], w the right singular vector of A's smallest singular value (np.linalg.svd, fp64).
With fewer than two views selected, X is NaN (the reference raises on 0 rows and returns an arbitrary point of the one ray
for 1 view); the selected count is returned with it.
"""
from __future__ import annotations

import numpy as np


def select_views(conf, conf_thres=0.05):
    """conf [V] scores of one joint -> the selected view indices, increasing (step 1, literally)."""
    conf = np.asarray(conf, dtype=np.float32)
    t = float(conf_thres)
    while True:
        sel = np.flatnonzero(conf > np.float32(t))
        if t < -1:
            break
        if len(sel) <= 1:
            t -= 0.05
        else:
            break
    return sel


def triangulate_one(pts, M, sel):
    """pts [V,2] float32 image px, M [V,3,4] fp64, sel the selected views -> (X [3], singular values of A, descending)."""
    if len(sel) < 2:
        return np.full(3, np.nan), np.full(4, np.nan)
    A = []
    for v in sel:
        x, y = np.float64(pts[v, 0]), np.float64(pts[v, 1])
        A.append(x * M[v, 2] - M[v, 0])
        A.append(y * M[v, 2] - M[v, 1])
    _, s, vt = np.linalg.svd(np.stack(A))
    return vt[-1, :3] / vt[-1, 3], s


def triangulate_loop(locs, scores, P, conf_thres=0.05):
    """The reference's shape: a loop over frames and joints.  locs [V,N,J,2], scores [V,N,J], P [V,N,3,4] ->
    (X [N,J,3] fp64, n_used [N,J] int32)."""
    locs, scores, P = np.asarray(locs, np.float32), np.asarray(scores, np.float32), np.asarray(P, np.float64)
    V, N, J = scores.shape
    X, n_used = np.zeros((N, J, 3)), np.zeros((N, J), np.int32)
    for n in range(N):
        for j in range(J):
            sel = select_views(scores[:, n, j], conf_thres)
            X[n, j] = triangulate_one(locs[:, n, j], P[:, n], sel)[0]
            n_used[n, j] = len(sel)
    return X, n_used


def selection_mask(scores, conf_thres=0.05):
    """step 1 for every problem at once: scores [V,...] -> bool mask [V,...].  Every problem starts at the same t and steps it
    alike, so one shared t sequence serves all; a problem stops at the first t where it selects two or more views, or t < -1."""
    scores = np.asarray(scores, dtype=np.float32)
    mask = np.zeros(scores.shape, bool)
    done = np.zeros(scores.shape[1:], bool)
    t = float(conf_thres)
    while not done.all():
        m = scores > np.float32(t)
        stop = ~done & ((m.sum(0) >= 2) | (t < -1))
        mask[:, stop] = m[:, stop]
        done |= stop
        if t < -1:
            break
        t -= 0.05
    return mask


def triangulate(locs, scores, P, conf_thres=0.05):
    """Steps 1-3 for a batch: locs [V,N,J,2], scores [V,N,J], P [V,N,3,4] -> (X [N,J,3] fp64, n_used [N,J] int32,
    singular values [N,J,4] of A, descending, NaN where fewer than two views are selected).  The SVDs of the problems that
    select the same number of views run as one stacked np.linalg.svd call, which is the same LAPACK routine per matrix as
    `triangulate_one` calls."""
    locs, scores, P = np.asarray(locs, np.float32), np.asarray(scores, np.float32), np.asarray(P, np.float64)
    V, N, J = scores.shape
    mask = selection_mask(scores, conf_thres).reshape(V, N * J).T               # [NJ, V]
    n_used = mask.sum(1)
    pts = locs.reshape(V, N * J, 2).transpose(1, 0, 2).astype(np.float64)       # [NJ, V, 2]
    M = np.repeat(P.transpose(1, 0, 2, 3), J, axis=0)                           # [NJ, V, 3, 4]
    X, sv = np.full((N * J, 3), np.nan), np.full((N * J, 4), np.nan)
    order = np.argsort(~mask, axis=1, kind="stable")                            # selected views first, increasing
    for k in np.unique(n_used[n_used >= 2]):
        idx = np.flatnonzero(n_used == k)
        views = order[idx, :k]                                                  # [B, k]
        p = np.take_along_axis(pts[idx], views[..., None], 1)                   # [B, k, 2]
        m = np.take_along_axis(M[idx], views[..., None, None], 1)               # [B, k, 3, 4]
        A = np.empty((len(idx), k, 2, 4))
        A[:, :, 0] = p[..., 0:1] * m[:, :, 2] - m[:, :, 0]
        A[:, :, 1] = p[..., 1:2] * m[:, :, 2] - m[:, :, 1]
        _, s, vt = np.linalg.svd(A.reshape(len(idx), 2 * k, 4))
        X[idx] = vt[:, -1, :3] / vt[:, -1, 3:]
        sv[idx] = s
    return X.reshape(N, J, 3), n_used.reshape(N, J).astype(np.int32), sv.reshape(N, J, 4)
