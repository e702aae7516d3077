"""CPU: the peak finder's numpy oracle against the reference function on non-finite, tied and degenerate heat-maps
(tests/golden/peaks_edges.npz, frozen by oracle/make_golden_peaks.py), and the peak finders' argument refusals, made without
a GPU: every refused call returns before anything is launched."""
import ctypes
import os
import re
import warnings

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build
from oracle import make_golden_peaks as mg
from oracle import peaks_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "peaks_edges.npz"))
EINVAL = -1
INT32_MAX = 2 ** 31 - 1


def assert_matches_golden(name, locs, score):
    """scores bit for bit (NaN and ±inf included); locations within 3e-4 image px, NaN exactly where the reference's are"""
    gl, gs = GOLD[name + "_locs"], GOLD[name + "_score"]
    assert locs.shape == gl.shape and score.shape == gs.shape
    np.testing.assert_array_equal(np.asarray(score, np.float32).view(np.uint32), gs.view(np.uint32))
    np.testing.assert_array_equal(np.isnan(locs), np.isnan(gl))
    np.testing.assert_allclose(locs, gl, rtol=0, atol=3e-4, equal_nan=True)


@pytest.mark.parametrize("name", sorted(mg.EDGES))
def test_oracle_matches_reference_golden(name):
    J, H, W, radius, ds, _ = mg.EDGES[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)                 # inf - inf and 0 · inf in the NaN cases
        locs, score = po.find_tensor_peak_batch(mg.edge_heatmaps(name), radius, ds)
    assert_matches_golden(name, locs, score)


def test_goldens_hold_the_edges():
    """the frozen table contains what it is meant to: NaN scores and locations, a finite score with a NaN location (0 · -inf),
    the all -inf map at index 0, and each tie resolved to its first index"""
    assert np.isnan(GOLD["nan_score"][:4]).all() and np.isnan(GOLD["nan_locs"][:4]).all()
    assert np.isfinite(GOLD["nan_locs"][4]).all()
    s, l = GOLD["inf_score"], GOLD["inf_locs"]
    assert s[0] == np.inf and np.isfinite(s[1]) and np.isnan(l[1]).all() and s[2] == -np.inf
    assert (l[2] == [1.5, 1.5]).all()                                   # index 0: pix2coord(0) = 4/2 - 0.5
    _, _, W, _, ds, _ = mg.EDGES["ties"]
    for j, idx in enumerate(mg.EDGE_JOINTS["ties"]):
        at = np.array([[i % W, i / W] for i in idx]) * ds + ds / 2 - 0.5   # each tied pixel's image position (true division)
        assert np.linalg.norm(at - GOLD["ties_locs"][j], axis=1).argmin() == 0
    assert str(GOLD["torch_version"]).split(".")[0] == "2"


# ---- argument refusals --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def header_max_r():
    src = open(os.path.join(ROOT, "include", "epipolar_b200.h")).read()
    return int(re.search(r"#define EPI_PEAKS_MAX_R (\d+)", src).group(1))


def test_max_r_is_the_int32_window_bound():
    """R = EPI_PEAKS_MAX_R is the largest R whose window loop, counting to (2R+1)^2 + 31, stays in int32"""
    R = header_max_r()
    assert R == _lib.PEAKS_MAX_R
    assert (2 * R + 1) ** 2 + 31 <= INT32_MAX < (2 * R + 3) ** 2 + 31


BAD_RADII = {"inf": (float("inf"), b"finite"), "nan": (float("nan"), b"bad shape or radius"),
             "-inf": (float("-inf"), b"bad shape or radius"), "1e30": (1e30, b"too large"),
             "R_max_plus_1": (_lib.PEAKS_MAX_R + 0.5, b"too large"), "R0": (0.49, b"at least 1")}


def call(lib, entry, radius=2.0, B=1, J=1, H=4, W=4):
    buf = (ctypes.c_float * 64)()
    a = ctypes.addressof(buf)
    if entry == "single":
        return lib.epi_find_peaks_f32(a, a, a, B, J, H, W, radius, 4.0, 1e-6, 0, None)
    return lib.epi_find_peaks_best_f32(a, a, a, None, 2, B, J, H, W, radius, 4.0, 1e-6, 0, None)


@pytest.mark.parametrize("entry", ["single", "best"])
@pytest.mark.parametrize("case", list(BAD_RADII))
def test_abi_refuses_radius(lib, entry, case):
    radius, msg = BAD_RADII[case]
    assert call(lib, entry, radius=radius) == EINVAL
    assert msg in lib.epi_last_error(), lib.epi_last_error()
    if case == "R_max_plus_1":
        assert str(_lib.PEAKS_MAX_R).encode() in lib.epi_last_error()


@pytest.mark.parametrize("entry", ["single", "best"])
def test_abi_refuses_bj_beyond_int32_warps(lib, entry):
    assert call(lib, entry, B=1 << 14, J=1 << 13) == EINVAL               # 2^27 warps > INT32_MAX / 32
    assert b"B * J too large" in lib.epi_last_error(), lib.epi_last_error()
    assert call(lib, entry, B=1 << 14, J=1 << 13, radius=float("inf")) == EINVAL
    assert call(lib, entry, B=0) == EINVAL and call(lib, entry, H=1) == EINVAL


def test_python_refusals():
    """find_tensor_peak_batch / _best raise ValueError on the same arguments, before they look at the device"""
    maps = {"batch": torch.zeros(2, 3, 8, 8), "best": torch.zeros(2, 2, 3, 8, 8)}
    calls = {"batch": epi.find_tensor_peak_batch, "best": epi.find_tensor_peak_best}
    for k, f in calls.items():
        for radius, msg in ((float("inf"), "not ok"), (float("nan"), "not ok"), (-1.0, "not ok"), (1e30, "too large"),
                            (_lib.PEAKS_MAX_R + 0.5, "too large")):
            with pytest.raises(ValueError, match=msg):
                f(maps[k], radius, 4.0)
        with pytest.raises(RuntimeError, match="no CPU implementation"):  # the largest R is accepted
            f(maps[k], _lib.PEAKS_MAX_R + 0.49, 4.0)
    big = torch.zeros(1, 1, 2, 2).expand(1 << 14, 1 << 13, 2, 2)          # B·J = 2^27 joints, no storage behind them
    with pytest.raises(ValueError, match="too large"):
        epi.find_tensor_peak_batch(big, 2.0, 4.0)
    with pytest.raises(ValueError, match="too large"):
        epi.find_tensor_peak_best(big[None], 2.0, 4.0)
