"""CPU: the pymvg-mode triangulation's numpy oracle (oracle/triangulate_oracle.py) on hand-built cases, and the C ABI's and the
Python entry point's refusals, checked without a GPU."""
import ctypes
import subprocess

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build
from epipolar_transformers_b200 import synthetic as syn
from oracle import triangulate_oracle as to

EINVAL = -1


def project(P, X):
    uv = P @ np.append(X, 1.0)
    return uv[..., :2] / uv[..., 2:3]


# ---- the oracle ------------------------------------------------------------------------------------------------------------------
def test_known_truth_float32_exact():
    """a 3-D point and integer cameras whose projections are float32-exact: recovered to 1e-9 relative from 2 and 3 views"""
    X = np.array([120.0, -80.0, 2000.0])
    P = np.array([[[500, 0, 256, 0], [0, 500, 256, 0], [0, 0, 1, 0]],
                  [[500, 0, 256, -500 * 400], [0, 500, 256, 0], [0, 0, 1, 0]],
                  [[500, 0, 256, 0], [0, 500, 256, -500 * 250], [0, 0, 1, 0]]], np.float64)
    pts = project(P, X)
    assert (pts.astype(np.float32) == pts).all()
    for V in (2, 3):
        Xt, s = to.triangulate_one(pts[:V].astype(np.float32), P[:V], np.arange(V))
        assert np.linalg.norm(Xt - X) <= 1e-9 * np.linalg.norm(X)
        b, n, _ = to.triangulate(pts[:V, None, None].astype(np.float32), np.ones((V, 1, 1), np.float32), P[:V, None])
        assert n[0, 0] == V and np.linalg.norm(b[0, 0] - X) <= 1e-9 * np.linalg.norm(X)


def test_threshold_compare_is_float32():
    """float32(0.05) > 0.05 is False in numpy's float32 compare: a score of exactly float32(0.05) is not selected"""
    c = np.array([np.float32(0.05), 0.9, 0.8, np.nextafter(np.float32(0.05), np.float32(1))], np.float32)
    assert list(to.select_views(c)) == [1, 2, 3]
    c[1:3] = 0.0
    assert list(to.select_views(c)) == [0, 3]                                   # one view above 0.05: relax to t = 0.0


def test_relaxation_picks_next_bin():
    """all scores under the threshold: t steps down by 0.05 until two views pass, and no further"""
    c = np.array([0.01, -0.02, -0.07, -0.30], np.float32)
    assert list(to.select_views(c)) == [0, 1]                                   # t = 0.05, 0.0 (one view), -0.05 (two)
    c = np.array([-0.12, -0.34, -0.36, -0.90], np.float32)
    assert list(to.select_views(c)) == [0, 1]                                   # ... -0.35 (two: -0.12, -0.34)


def test_relaxation_past_minus_one():
    """t stepped in fp64 from 0.05 reaches -1.0000000000000002 after 21 steps: that pass is the last, at float32 -1.0, and it
    keeps what it selects, two or more views or fewer (a t stepped without rounding would go on to -1.05)"""
    t = 0.05
    for _ in range(21):
        t -= 0.05
    assert t < -1 and np.float32(t) == -1.0
    c = np.array([-0.99, -0.999, -5.0, np.nan], np.float32)
    assert list(to.select_views(c)) == [0, 1]
    c = np.array([-0.99, -1.0, -5.0, -3.0], np.float32)
    assert list(to.select_views(c)) == [0]


def test_nan_scores_never_selected():
    c = np.array([np.nan, 0.5, np.nan, 0.7], np.float32)
    assert list(to.select_views(c)) == [1, 3]
    c = np.full(4, np.nan, np.float32)
    assert list(to.select_views(c)) == []


@pytest.mark.parametrize("scores,count", [([-3.0, -3.0, -3.0], 0), ([0.9, -3.0, -3.0], 1)])
def test_zero_and_one_views_give_nan(scores, count):
    V = len(scores)
    P = syn.ring_cameras(V, 256)[:, None]
    locs = np.full((V, 1, 1, 2), 100.0, np.float32)
    X, n, sv = to.triangulate(locs, np.array(scores, np.float32)[:, None, None], P)
    assert n[0, 0] == count and np.isnan(X).all() and np.isnan(sv).all()
    Xl, nl = to.triangulate_loop(locs, np.array(scores, np.float32)[:, None, None], P)
    assert nl[0, 0] == count and np.isnan(Xl).all()


def test_batched_oracle_equals_loop():
    """the stacked form (`triangulate`) gives the loop's (`triangulate_loop`) counts and points bit for bit"""
    rng = np.random.default_rng(5)
    V, N, J = 5, 6, 17
    P = np.stack([syn.ring_cameras(V, 256, jitter=20.0, seed=n) for n in range(N)], 1)
    locs = rng.uniform(0, 256, (V, N, J, 2)).astype(np.float32)
    scores = rng.choice([-1.3, -0.6, -0.2, 0.0, 0.03, 0.05, 0.2, np.nan], (V, N, J)).astype(np.float32)
    scores += rng.uniform(-0.02, 0.02, scores.shape).astype(np.float32)
    a, na, _ = to.triangulate(locs, scores, P)
    b, nb = to.triangulate_loop(locs, scores, P)
    assert (na == nb).all() and len(np.unique(na)) >= 4
    assert np.array_equal(a, b, equal_nan=True)


# ---- the C ABI -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_probe_and_dtype(lib):
    assert lib.epi_triangulate() == 1
    assert _lib.EPI_DTYPE_F64 == 3


REFUSALS = {
    "null_locs": b"must be non-null", "null_scores": b"must be non-null", "null_P": b"must be non-null",
    "null_X": b"must be non-null", "null_n": b"must be non-null", "V1": b"V must be in [2, 64]", "V65": b"V must be in [2, 64]",
    "N0": b"N >= 1", "J0": b"J >= 1", "NJ": b"2^31 - 1", "dtype_bf16": b"P_dtype", "dtype_9": b"P_dtype",
    "conf_nan": b"conf_thres must be finite", "conf_inf": b"conf_thres must be finite", "conf_big": b"<= 1000",
    "locs_misaligned": b"aligned", "P64_misaligned": b"aligned",
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_abi_refusals(lib, case):
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)
    args = dict(locs=a, scores=a, P=a, dtype=_lib.EPI_DTYPE_F32, conf=0.05, V=4, N=2, J=17, X=a, n=a)
    key = case.split("_")[1] if case.startswith("null_") else None
    if key:
        args[key] = None
    elif case == "V1":
        args["V"] = 1
    elif case == "V65":
        args["V"] = 65
    elif case == "N0":
        args["N"] = 0
    elif case == "J0":
        args["J"] = 0
    elif case == "NJ":
        args["N"], args["J"] = 65536, 32768
    elif case == "dtype_bf16":
        args["dtype"] = _lib.EPI_DTYPE_BF16
    elif case == "dtype_9":
        args["dtype"] = 9
    elif case == "conf_nan":
        args["conf"] = float("nan")
    elif case == "conf_inf":
        args["conf"] = float("-inf")
    elif case == "conf_big":
        args["conf"] = 1000.5
    elif case == "locs_misaligned":
        args["locs"] = a + 4
    elif case == "P64_misaligned":
        args["P"], args["dtype"] = a + 4, _lib.EPI_DTYPE_F64
    rc = lib.epi_triangulate_dlt_f64(args["locs"], args["scores"], args["P"], args["dtype"], args["conf"], args["V"], args["N"],
                                     args["J"], args["X"], args["n"], None)
    assert rc == EINVAL
    assert REFUSALS[case] in lib.epi_last_error(), lib.epi_last_error()


# ---- Python --------------------------------------------------------------------------------------------------------------------
def test_python_refusals():
    l, s, P = torch.zeros(4, 2, 17, 2), torch.zeros(4, 2, 17), torch.zeros(4, 2, 3, 4)
    with pytest.raises(ValueError, match=r"locs must be \[V,N,J,2\]"):
        epi.triangulate_views(l[..., :1], s, P)
    with pytest.raises(ValueError, match="scores must be"):
        epi.triangulate_views(l, s[:, :1], P)
    with pytest.raises(ValueError, match="P must be"):
        epi.triangulate_views(l, s, P[..., :3])
    with pytest.raises(ValueError, match="2 to 64 views"):
        epi.triangulate_views(l[:1], s[:1], P[:1])
    with pytest.raises(ValueError, match="2 to 64 views"):
        epi.triangulate_views(torch.zeros(65, 1, 1, 2), torch.zeros(65, 1, 1), torch.zeros(65, 1, 3, 4))
    with pytest.raises(ValueError, match="floating-point"):
        epi.triangulate_views(l, s.int(), P)
    with pytest.raises(ValueError, match="conf_thres"):
        epi.triangulate_views(l, s, P, conf_thres=float("nan"))
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        epi.triangulate_views(l, s, P)


def test_library_without_triangulation(monkeypatch, tmp_path):
    """the triangulation entry points are new symbols: a library without them still loads, and a triangulate_views call names
    the missing probe"""
    old = [s for s in _lib.EXPORTS if s not in _lib.TRIANGULATE_EXPORTS]
    assert len(old) == len(_lib.EXPORTS) - 2
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    _lib.load()
    with pytest.raises(RuntimeError, match="epi_triangulate.*cannot triangulate"):
        epi.triangulate_views(torch.zeros(4, 2, 17, 2), torch.zeros(4, 2, 17), torch.zeros(4, 2, 3, 4))
