"""TEST INFRASTRUCTURE — freezes outputs of the UNMODIFIED reference find_tensor_peak_batch
(/root/reference/modeling/backbones/basic_batch.py:17-63) as tests/golden/peaks.npz (smooth maps, `CASES`) and
tests/golden/peaks_edges.npz (non-finite, tied and degenerate maps, `EDGES`).  Build container only.
    python -m oracle.make_golden_peaks
Inputs are regenerated from seeds by `heatmaps(name)` and `edge_heatmaps(name)` (also used by the tests)."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {   # name: (J, H, W, radius, downsample, kind)
    "h36m_r50": (17, 64, 64, 8.0, 4.0, "gauss"),            # KEYPOINT.SIGMA = 8 (keypoint_h36m_zresidual_fixed.yaml:40)
    "r152_384": (17, 96, 96, 8.0, 4.0, "gauss"),
    "small_radius": (5, 20, 28, 2.0, 8.0, "gauss"),
    "border": (6, 16, 16, 3.0, 4.0, "border"),              # peaks on the map border: zero padding of the window
    "noise": (8, 24, 24, 4.0, 4.0, "noise"),
}


def heatmaps(name):
    J, H, W, radius, ds, kind = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.zeros((J, H, W), np.float32)
    for j in range(J):
        if kind == "border":
            cx, cy = [(0.0, 0.0), (W - 1.0, 0.3), (0.4, H - 1.0), (W - 1.0, H - 1.0), (W / 2, 0.0), (0.0, H / 2)][j % 6]
        else:
            cx, cy = rng.uniform(2, W - 3), rng.uniform(2, H - 3)
        g = np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * (1.0 + 0.25 * radius) ** 2))
        if kind == "noise":
            g = 0.2 * g + rng.random((H, W)) * 0.3
        else:
            g = g + 0.01 * rng.standard_normal((H, W))
        out[j] = g.astype(np.float32)
    return out


# Edge cases: name -> (J, H, W, radius, downsample, kind).  Every joint of a case is a smooth bump plus noise, then
# `edge_heatmaps` applies the kind's per-joint change (EDGE_JOINTS).  The reference's own float32 arithmetic is what
# is frozen, NaN included: torch.max returns the first NaN and F.threshold keeps NaN, so a map holding a NaN has a NaN score
# and (through the window's bilinear samples) a NaN location.
EDGES = {
    "nan": (5, 16, 20, 2.0, 4.0, "nan"),
    "inf": (6, 16, 17, 2.0, 4.0, "inf"),                   # W - 1 = 16: the window's middle column samples x = 8 exactly
    "ties": (5, 12, 16, 2.0, 4.0, "ties"),
    "radius_0p5": (4, 16, 20, 0.5, 4.0, "bump"),           # R = 1, step 0.5
    "radius_1p49": (4, 16, 20, 1.49, 4.0, "bump"),         # R = 1, step 1.49
    "radius_2p5": (4, 16, 20, 2.5, 4.0, "bump"),           # R = 3, step 5/6
    "radius_2p6": (4, 16, 20, 2.6, 4.0, "bump"),           # R = 3, step 2.6/3
    "radius_40": (4, 16, 20, 40.0, 4.0, "bump"),           # window far larger than the map
    "map_2x2": (4, 2, 2, 2.0, 4.0, "noise"),
    "map_2x37": (4, 2, 37, 2.0, 4.0, "noise"),
    "map_37x2": (4, 37, 2, 2.0, 4.0, "noise"),
    "map_13x200": (4, 13, 200, 3.0, 4.0, "bump"),
    "map_96x72": (4, 96, 72, 8.0, 4.0, "bump"),
    "ds_1": (4, 16, 20, 2.0, 1.0, "bump"),
    "ds_8": (4, 16, 20, 2.0, 8.0, "bump"),
    "ds_0p25": (4, 16, 20, 2.0, 0.25, "bump"),
}
EDGE_JOINTS = {
    "nan": ["NaN away from the max", "NaN at the max", "three NaNs", "NaN next to the max", "finite"],
    "inf": ["+inf at the max", "-inf next to the max", "all -inf", "constant", "all negative", "finite"],
    # flat indices of exactly tied maxima; the first sits in a higher warp lane (index % 32) than a later one
    "ties": [(2, 33), (31, 32), (5, 100), (0, 191), (7, 38, 69)],
}


def edge_heatmaps(name):
    J, H, W, radius, ds, kind = EDGES[name]
    rng = np.random.default_rng(sum(map(ord, name)) + 1000)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.zeros((J, H, W), np.float32)
    for j in range(J):
        cx, cy = rng.uniform(0, W - 1), rng.uniform(0, H - 1)
        what = EDGE_JOINTS[kind][j] if kind in EDGE_JOINTS else None
        if what == "-inf next to the max":
            cx = 8.0            # max in column 8 of 17: the middle column's taps are x = 8 (weight 1) and x = 9 (weight 0)
        g = np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * 1.5 ** 2))
        if kind in ("noise", "ties"):
            g = 0.2 * g + rng.random((H, W)) * 0.3
        else:
            g = g + 0.01 * rng.standard_normal((H, W))
        m = g.astype(np.float32)
        at = int(np.argmax(m))
        y, x = divmod(at, W)
        nxt = y * W + (x + 1 if x + 1 < W else x - 1)                # a neighbour of the max in the same row
        flat = m.reshape(-1)
        if what == "NaN away from the max":
            flat[(at + H * W // 2) % (H * W)] = np.nan
        elif what == "NaN at the max":
            flat[at] = np.nan
        elif what == "three NaNs":
            flat[[(at + 7) % (H * W), 3, (at + H * W - 9) % (H * W)]] = np.nan
        elif what == "NaN next to the max":
            flat[nxt] = np.nan
        elif what == "+inf at the max":
            flat[at] = np.inf
        elif what == "-inf next to the max":
            assert (W, x) == (17, 8), (W, x)
            flat[nxt] = -np.inf                                      # 0 · -inf = NaN in the zero-weight tap
        elif what == "all -inf":
            flat[:] = -np.inf
        elif what == "constant":
            flat[:] = 0.25
        elif what == "all negative":
            flat -= 2.0
        elif kind == "ties":
            flat[list(what)] = 1.0                                   # above every noise value (< 0.5)
        out[j] = m
    return out


def _reference_peaks():
    from oracle.make_golden_dropin import import_reference_resnet
    import importlib
    import_reference_resnet()
    return importlib.import_module("modeling.backbones.basic_batch").find_tensor_peak_batch


def main():
    import torch
    find = _reference_peaks()
    for table, maps, fname in ((CASES, heatmaps, "peaks.npz"), (EDGES, edge_heatmaps, "peaks_edges.npz")):
        rec = {}
        for name, (J, H, W, radius, ds, kind) in table.items():
            locs, score = find(torch.from_numpy(maps(name)), radius, ds)
            rec[name + "_locs"] = locs.numpy(); rec[name + "_score"] = score.numpy()
            print(name, locs[:2].numpy().round(3).tolist())
        rec["torch_version"] = np.array(torch.__version__)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", fname), **rec)


if __name__ == "__main__":
    main()
