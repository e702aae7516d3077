"""TEST INFRASTRUCTURE — numpy restatement of find_tensor_peak_batch
(/root/reference/modeling/backbones/basic_batch.py:17-63) in float64/float32, pinned to vectors frozen from the
reference itself by oracle/make_golden_peaks.py (tests/golden/peaks.npz).  NOT product code."""
from __future__ import annotations

import numpy as np


def find_tensor_peak_batch(heatmap, radius, downsample, threshold=0.000001, int_div=False, dtype=np.float32, window=False):
    """heatmap [J,H,W] -> (locs [J,2], score [J]), and with window=True also the thresholded window sub [J,S,S].

    Non-finite values follow the reference: the arg-max is the first NaN if there is one (torch.max), the threshold keeps
    NaN (F.threshold zeroes only v <= threshold), and a zero bilinear weight times ±inf is NaN."""
    heatmap = np.asarray(heatmap, dtype)
    J, H, W = heatmap.shape
    flat = heatmap.reshape(J, -1)
    index = flat.argmax(1)                                                   # first NaN, else first maximum (:24)
    score = flat[np.arange(J), index]
    index_w = (index % W).astype(dtype)                                      # :25
    index_h = (index // W).astype(dtype) if int_div else (index.astype(dtype) / dtype(W))   # :26 (true division in torch >= 1.5)
    norm = lambda x, L: dtype(-1.0) + dtype(2.0) * x / dtype(L - 1)          # :28-29
    b0, b1 = norm(index_w - dtype(radius), W), norm(index_h - dtype(radius), H)
    b2, b3 = norm(index_w + dtype(radius), W), norm(index_h + dtype(radius), H)
    R = int(radius + 0.5)                                                    # :40
    S = 2 * R + 1
    base = (dtype(2.0) * np.arange(S, dtype=dtype) + dtype(1.0)) / dtype(S) - dtype(1.0)      # affine_grid, align_corners=False
    gx = ((b2 - b0) / dtype(2))[:, None] * base[None, :] + ((b2 + b0) / dtype(2))[:, None]    # [J,S]
    gy = ((b3 - b1) / dtype(2))[:, None] * base[None, :] + ((b3 + b1) / dtype(2))[:, None]
    px = ((gx + dtype(1)) * dtype(W) - dtype(1)) / dtype(2)                  # grid_sample unnormalise, align_corners=False
    py = ((gy + dtype(1)) * dtype(H) - dtype(1)) / dtype(2)
    x0 = np.floor(px).astype(np.int64); y0 = np.floor(py).astype(np.int64)
    wx = px - x0; wy = py - y0
    sub = np.zeros((J, S, S), dtype)
    for dy, wyy in ((0, 1 - wy), (1, wy)):
        for dx, wxx in ((0, 1 - wx), (1, wx)):
            yy = y0 + dy; xx = x0 + dx                                       # [J,S]
            inb = ((yy >= 0) & (yy < H))[:, :, None] & ((xx >= 0) & (xx < W))[:, None, :]
            v = heatmap[np.arange(J)[:, None, None], np.clip(yy, 0, H - 1)[:, :, None], np.clip(xx, 0, W - 1)[:, None, :]]
            sub += np.where(inb, v, dtype(0)) * (wyy[:, :, None] * wxx[:, None, :]).astype(dtype)
    sub = np.where(sub <= dtype(threshold), dtype(0), sub)                   # F.threshold keeps NaN (:50)
    X = (dtype(-radius) + dtype(radius * 1.0 / R) * np.arange(S, dtype=dtype))                # arange(-r, r+1e-4, r/R) (:52-53)
    sum_region = sub.reshape(J, -1).sum(1) + dtype(np.finfo(float).eps)
    x = (sub * X[None, None, :]).reshape(J, -1).sum(1) / sum_region + index_w
    y = (sub * X[None, :, None]).reshape(J, -1).sum(1) / sum_region + index_h
    p2c = lambda v: v * dtype(downsample) + dtype(downsample / 2.0) - dtype(0.5)              # vision/multiview.py:154-157
    locs = np.stack([p2c(x), p2c(y)], 1)
    return (locs, score, sub) if window else (locs, score)
