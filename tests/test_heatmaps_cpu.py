"""CPU: the heat-map forward (EpiHeadParams, epi_fusion_heatmaps_*, epi_fold_head_f32) and its Python entry points, checked
without a GPU: struct layout, argument refusals, workspace and cache sizes, Python refusals, loading a library built before the
entry points, and the fold's arithmetic against numpy in fp64 (on the GPU when there is one)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build
from tests.test_view_sources_cpu import pipe_cache, pipe_workspace, tbl
from tests.test_views_cpu import C, H, W, _cfg2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")
EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_head_params_layout_matches_header():
    fields = ["A", "B", "b", "heat", "heat_stride", "J", "reserved"]
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "off.c")
        open(c, "w").write('#include <stdio.h>\n#include "%s"\nint main(){printf("%s %%zu", %s, sizeof(EpiHeadParams));return 0;}' % (
            HEADER, " ".join(["%zu"] * len(fields)), ", ".join("__builtin_offsetof(EpiHeadParams, %s)" % f for f in fields)))
        exe = os.path.join(d, "off")
        subprocess.check_call(["gcc", c, "-o", exe])
        got = list(map(int, subprocess.check_output([exe]).split()))
    P = _lib.EpiHeadParams
    assert got == [getattr(P, f).offset for f in fields] + [ctypes.sizeof(P)]


def pair_params():
    buf = (ctypes.c_float * 64)()
    addr = ctypes.addressof(buf)
    p = _lib.EpiFusionParams()
    p.feat_ref = p.feat_src = p.P_ref = p.P_src = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 8
    p.downsample = 4.0; p.img_scale = 1.0
    h = _lib.EpiHeadParams()
    h.A = h.b = h.heat = addr
    h.J = 17
    return p, h, buf


REFUSALS = {
    "out": b"out must be null", "z": b"z_weight_folded must be null", "add_ref": b"add_ref_residual must be 0",
    "null_head": b"head params are null", "null_A": b"non-null", "null_heat": b"non-null", "J0": b"J must be",
    "J65": b"J must be", "reserved": b"reserved", "heat_misaligned": b"aligned", "n_views_1": b"n_views",
    "bad_table": b"not a view", "no_P": b"P_ref/P_src required",
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_abi_refusals(lib, case):
    p, h, buf = pair_params()
    addr = ctypes.addressof(buf)
    ptr, S = None, 0
    if case == "out":
        p.out = addr
    elif case == "z":
        p.z_weight_folded = p.z_bias_folded = addr
    elif case == "add_ref":
        p.add_ref_residual = 1
    elif case == "null_A":
        h.A = None
    elif case == "null_heat":
        h.heat = None
    elif case == "J0":
        h.J = 0
    elif case == "J65":
        h.J = 65
    elif case == "reserved":
        h.reserved[1] = 1
    elif case == "heat_misaligned":
        h.heat = addr + 2
    elif case == "n_views_1":
        p.n_views = 1
    elif case == "bad_table":
        p.feat_src = p.P_src = None
        p.n_views = 3
        ptr, S, _t = tbl([[1], [3], [0]])
    elif case == "no_P":
        p.P_src = None
    hp = None if case == "null_head" else ctypes.byref(h)
    assert lib.epi_fusion_heatmaps_f32(ctypes.byref(p), hp, ptr, S, None) == EINVAL
    assert REFUSALS[case] in lib.epi_last_error(), lib.epi_last_error()


def test_fold_refusals(lib):
    buf = (ctypes.c_float * 4)()
    a = ctypes.addressof(buf)
    assert lib.epi_fold_head_f32(None, None, None, None, 0, 1, 1, a, a, None) == EINVAL
    assert lib.epi_fold_head_f32(a, None, None, None, 0, 0, 1, a, a, None) == EINVAL
    assert b"J >= 1" in lib.epi_last_error()


def test_probe(lib):
    assert lib.epi_fusion_heatmaps() == 1


# ---- sizes: the plan of the call without a head that stores a pixel-major fp32 plane (no z GEMM planes) ------------------------
@pytest.mark.parametrize("V,S,N", [(2, 1, 1), (4, 1, 4), (4, 2, 2)])
@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("cache", [True, False], ids=["cache", "nocache"])
def test_sizes_match_formula(lib, V, S, N, dtype, cache):
    p = _cfg2(V, N, dtype, z=False, cache=cache)
    h = _lib.EpiHeadParams()
    h.J = 17
    ptr, S_, _t = tbl([[(v + 1 + j) % V for j in range(S)] for v in range(V)])
    lo = dtype != _lib.EPI_DTYPE_BF16
    assert lib.epi_fusion_heatmaps_workspace_bytes(ctypes.byref(p), ctypes.byref(h), ptr, S_) == pipe_workspace(V, S, N, lo, False, cache)
    assert lib.epi_fusion_heatmaps_cache_bytes(ctypes.byref(p), ctypes.byref(h), ptr, S_) == pipe_cache(V, S, N)
    # no table: the all-others views form sizes, as the call without a head with a misaligned `out` plans them
    q = _cfg2(V, N, dtype, z=False, cache=cache)
    q.out = 4
    assert lib.epi_fusion_heatmaps_workspace_bytes(ctypes.byref(q), ctypes.byref(h), None, 0) == lib.epi_fusion_workspace_bytes(ctypes.byref(q))
    h.J = 65
    assert lib.epi_fusion_heatmaps_workspace_bytes(ctypes.byref(p), ctypes.byref(h), ptr, S_) == 0
    assert lib.epi_fusion_heatmaps_workspace_bytes(ctypes.byref(p), None, ptr, S_) == 0


# ---- Python ------------------------------------------------------------------------------------------------------------------
def test_python_refusals():
    conv = torch.nn.Conv2d(8, 17, 1)
    with pytest.raises(ValueError, match="1x1"):
        epi.head_weights(torch.nn.Conv2d(8, 17, 3))
    with pytest.raises(ValueError, match="1 to 64"):
        epi.head_weights((torch.zeros(65, 8), None))
    with pytest.raises(ValueError, match=r"\[J\]"):
        epi.head_weights((torch.zeros(17, 8), torch.zeros(3)))
    w, b = epi.head_weights(conv)
    assert w.shape == (17, 8) and b is conv.bias
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        epi.fold_head(w, b)
    f, P = torch.zeros(4, 1, 8, 8, 8), torch.zeros(4, 1, 3, 4)
    for call in (lambda: epi.standard_views_test(None, torch.nn.ReLU(), f, P, [[1], [2], [3], [0]], 2.0, 4.0, fuse_head=True),
                 lambda: epi.multitest_views(None, torch.nn.Conv2d(8, 17, 3), f, P, 2.0, 4.0, fuse_head=True),
                 lambda: epi.multitest(None, torch.nn.Sequential(conv), f[0], f[1:], P[0], P[1:], 2.0, 4.0, fuse_head=True)):
        with pytest.raises(ValueError, match="1x1"):
            call()
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(8, 8), NFEATS=8), EPIPOLAR=dict(SAMPLESIZE=8, PARAMETERIZED=("z",)))
    m = epi.Epipolar(cfg=cfg)
    with pytest.raises(RuntimeError, match="eval"):
        m.train().forward_heatmaps(f[0], f[1], P[0], P[1], conv)
    with pytest.raises(RuntimeError, match="inference only"):
        m.eval().forward_heatmaps(f[0], f[1], P[0], P[1], conv)             # conv.weight requires grad under grad mode
    with torch.no_grad(), pytest.raises(ValueError, match="takes 8 channels"):
        m.forward_heatmaps(f[0, :, :4], f[1, :, :4], P[0], P[1], conv)


def test_load_accepts_library_without_heatmaps(monkeypatch, tmp_path):
    """the heat-map entry points are new symbols: a library without them still loads and runs every other form, and a call with
    a head names the missing probe"""
    old = [s for s in _lib.EXPORTS if s not in _lib.HEATMAPS_EXPORTS]
    assert len(old) == len(_lib.EXPORTS) - 5
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    _lib.load()
    f, P = torch.zeros(2, 8, 8, 8), torch.zeros(2, 3, 4)
    with pytest.raises(RuntimeError, match="epi_fusion_heatmaps"):
        epi.epipolar_fusion(f, f, P, P, K=8, head=torch.nn.Conv2d(8, 17, 1))
    with pytest.raises(RuntimeError, match="epi_fold_head_f32"):
        epi.fold_head(torch.zeros(17, 8))
    with pytest.raises(RuntimeError, match="no CPU implementation"):           # a call without a head goes on to its own checks
        epi.epipolar_fusion(f, f, P, P, K=8)


@pytest.mark.skipif(not torch.cuda.is_available(), reason="the fold runs on the GPU")
@pytest.mark.parametrize("z", ["zres", "z", "noz"])
def test_fold_against_numpy_fp64(z):
    rng = np.random.default_rng(0)
    J, Cc = 17, 264
    Wh, bh = rng.standard_normal((J, Cc)).astype(np.float32), rng.standard_normal(J).astype(np.float32)
    Wf, bf = rng.standard_normal((Cc, Cc)).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    t = lambda a: torch.from_numpy(a).cuda()
    A, b = epi.fold_head(t(Wh), t(bh), None if z == "noz" else (t(Wf), t(bf)), z == "zres")
    d = lambda a: a.astype(np.float64)
    if z == "noz":
        A64, b64 = d(Wh), d(bh)
    else:
        A64 = d(Wh) @ (d(Wf) + (np.eye(Cc) if z == "zres" else 0))
        b64 = d(Wh) @ d(bf) + d(bh)
    assert (A.cpu().numpy() == A64.astype(np.float32)).all() and (b.cpu().numpy() == b64.astype(np.float32)).all()
