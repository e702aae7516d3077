"""CPU: the views form with a caller's source table (epi_fusion_view_sources_*) and its Python entry points, checked without a
GPU: table refusals, workspace and cache sizes, Python errors, and loading a library built before the entry points."""
import ctypes
import subprocess

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build, multiview
from epipolar_transformers_b200 import synthetic as syn
from tests.test_views_cpu import MAP1, PX, REC_BYTES, _cfg2, _views_params, al

EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def tbl(rows):
    t = np.ascontiguousarray(rows, dtype=np.int32)
    return t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), t.shape[1], t        # keep `t` alive with the pointer


# ---- ABI refusals (EPI_EINVAL before any CUDA call) ------------------------------------------------------------------------
REFUSALS = {
    "null_table": (None, b"null"),
    "s_zero": ("s0", b"S"),
    "entry_negative": ([[1], [-1], [0]], b"not a view"),
    "entry_too_large": ([[1], [3], [0]], b"not a view"),
    "self_pair": ([[1], [1], [0]], b"itself"),
    "n_views_0": ("n_views_0", b"n_views"),
    "n_src_2": ("n_src_2", b"n_src"),
    "feat_src": ("feat_src", b"must be null"),
    "P_src": ("P_src", b"must be null"),
    "too_many_entries": ("entries", b"EPI_VIEW_SOURCES_MAX"),
    "too_many_pairs": ("pairs", b"65535"),
}


def _refused(case):
    p, buf = _views_params(3)
    addr = ctypes.addressof(buf)
    rows, _ = REFUSALS[case]
    ptr, S, t = tbl([[1], [2], [0]])
    if rows is None:
        ptr = None
    elif rows == "s0":
        S = 0
    elif rows == "n_views_0":
        p.n_views = 0
    elif rows == "n_src_2":
        p.n_src = 2
    elif rows == "feat_src":
        p.feat_src = addr
    elif rows == "P_src":
        p.P_src = addr
    elif rows == "entries":                                      # 17 views · 16 sources = 272 > 256 entries
        p.n_views = 17
        ptr, S, t = tbl([[(v + 1 + j) % 17 for j in range(16)] for v in range(17)])
    elif rows == "pairs":                                        # 3·2·11000 pairs > 65535
        p.N = 11000
        ptr, S, t = tbl([[1, 2], [2, 0], [0, 1]])
    else:
        ptr, S, t = tbl(rows)
    return p, buf, ptr, S, t


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_abi_refusals(lib, case):
    p, _buf, ptr, S, _t = _refused(case)
    assert lib.epi_fusion_view_sources_forward_f32(ctypes.byref(p), ptr, S, None) == EINVAL
    msg = lib.epi_last_error()
    assert REFUSALS[case][1] in msg, msg


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_size_queries_answer_zero_for_unplannable_tables(lib, case):
    p, _buf, ptr, S, _t = _refused(case)
    if case in ("feat_src", "P_src"):
        pytest.skip("pointers do not change a plan's sizes (the call itself refuses them)")
    assert lib.epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), ptr, S) == 0
    assert lib.epi_fusion_view_sources_cache_bytes(ctypes.byref(p), ptr, S) == 0


def test_probe(lib):
    assert lib.epi_fusion_view_sources() == 1
    assert _lib.EPI_VIEW_SOURCES_MAX == 256


# ---- workspace and cache sizes: V·N staged view items, V·S·N pairs ---------------------------------------------------------
def pipe_workspace(V, S, N, lo, z, cache):
    NR, NP = V * N, V * S * N
    b = al(NR * MAP1 if lo else NR * MAP1 // 2) + NP * MAP1 + 256
    if z:
        b += 2 * 256 * 256 * 2
    if not cache:
        b += al(NP * PX * 2) + al(NP * 44)
    return b


def pipe_cache(V, S, N):
    NP = V * S * N
    records = NP * ((PX + 31) // 32) + V * S * (256 + N)
    return al(NP * 128) + al(NP * 44) + al(NP * PX * 2) + al(records * REC_BYTES)


@pytest.mark.parametrize("V,S,N", [(2, 1, 1), (4, 1, 1), (4, 1, 4), (4, 2, 2), (5, 3, 2), (4, 5, 1)])
@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16, _lib.EPI_DTYPE_F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("z", [True, False], ids=["z", "noz"])
@pytest.mark.parametrize("cache", [True, False], ids=["cache", "nocache"])
def test_pipe_sizes_match_formula(lib, V, S, N, dtype, z, cache):
    p = _cfg2(V, N, dtype, z, cache)
    ptr, S_, _t = tbl([[(v + 1 + j) % V if (v + 1 + j) % V != v else (v + 1) % V for j in range(S)] for v in range(V)])
    lo = dtype != _lib.EPI_DTYPE_BF16
    assert lib.epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), ptr, S_) == pipe_workspace(V, S, N, lo, z, cache)
    assert lib.epi_fusion_view_sources_cache_bytes(ctypes.byref(p), ptr, S_) == pipe_cache(V, S, N)


@pytest.mark.parametrize("V", [2, 3, 5])
def test_all_others_table_sizes_equal_views_form(lib, V):
    for variant in (_lib.EPI_VARIANT_AUTO, _lib.EPI_VARIANT_WARP, _lib.EPI_VARIANT_SECTOR):
        p = _cfg2(V, 2)
        p.variant = variant
        ptr, S, _t = tbl([[j + (j >= v) for j in range(V - 1)] for v in range(V)])
        assert lib.epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), ptr, S) == lib.epi_fusion_workspace_bytes(ctypes.byref(p))
        assert lib.epi_fusion_view_sources_cache_bytes(ctypes.byref(p), ptr, S) == lib.epi_fusion_cache_bytes(ctypes.byref(p))


# ---- the Python entry points -----------------------------------------------------------------------------------------------
def test_python_refusals():
    f = torch.zeros(3, 2, 8, 8, 8)
    P = torch.zeros(3, 2, 3, 4)
    with pytest.raises(ValueError, match=r"\[V,S\]"):
        epi.epipolar_fusion_views(f, P, K=8, sources=[1, 2, 0])
    with pytest.raises(ValueError, match=r"\[V,S\]"):
        epi.epipolar_fusion_views(f, P, K=8, sources=[[1], [2]])
    with pytest.raises(ValueError, match="itself"):
        epi.epipolar_fusion_views(f, P, K=8, sources=[[1], [1], [0]])
    with pytest.raises(ValueError, match=r"\[0, 3\)"):
        epi.epipolar_fusion_views(f, P, K=8, sources=np.array([[1], [3], [0]]))
    with pytest.raises(TypeError, match="integer"):
        epi.epipolar_fusion_views(f, P, K=8, sources=torch.tensor([[1.0], [2.0], [0.0]]))
    with pytest.raises(ValueError, match=r"sample_locs_in must be \[K,V,S,N,H,W,2\]"):
        epi.epipolar_fusion_views(f, P, K=8, sources=[[1], [2], [0]], sample_locs_in=torch.zeros(8, 3, 2, 2, 8, 8, 2))
    with pytest.raises(ValueError, match=r"out must be a \[V,S,N,C,H,W\]"):
        epi.epipolar_fusion_views(f, P, K=8, sources=[[1], [2], [0]], out=torch.zeros(3, 2, 2, 8, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU implementation"):   # a valid table with CPU maps is still refused
        epi.epipolar_fusion_views(f, P, K=8, sources=torch.tensor([[1], [2], [0]]))
    with pytest.raises(ValueError, match="one source"):
        epi.standard_views_test(None, None, f, P, [[1, 2], [2, 0], [0, 1]], 2.0, 4.0)


@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA tensor")
def test_cuda_table_refused():
    with pytest.raises(TypeError, match="synchronise"):
        epi.view_source_table(torch.tensor([[1], [0]], device="cuda"), 2)


def test_cuda_table_refused_without_gpu(monkeypatch):
    """a table that says it lives on the GPU is refused before anything reads it"""
    t = torch.tensor([[1], [0]])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(TypeError, match="synchronise"):
        epi.view_source_table(t, 2)


def test_view_source_table_accepts_lists_arrays_and_cpu_tensors():
    want = np.array([[1, 2], [2, 0], [0, 0]], dtype=np.int32)
    for s in (want.tolist(), want.astype(np.int64), torch.from_numpy(want.astype(np.int64)), torch.from_numpy(want)):
        got = epi.view_source_table(s, 3)
        assert got.dtype == np.int32 and got.flags.c_contiguous and (got == want).all()


def test_nearest_view_table():
    KRT = syn.ring_cameras(8, 256)
    t1 = multiview.nearest_view_table(KRT)
    t3 = multiview.nearest_view_table(torch.from_numpy(KRT), topk=3)
    assert t1.shape == (8, 1) and t3.shape == (8, 3) and t1.dtype == np.int32
    assert (t3[:, :1] == t1).all() and (t3 != np.arange(8)[:, None]).all()
    assert all(abs(int(s) - v) in (1, 7) for v, s in enumerate(t1[:, 0]))      # ring neighbours
    from epipolar_transformers_b200.distributed import source_view_table
    assert (source_view_table(KRT) == t1[:, 0]).all()
    with pytest.raises(ValueError, match="topk"):
        multiview.nearest_view_table(KRT, topk=8)


# ---- a library built before the source-table entry points ------------------------------------------------------------------
def test_load_accepts_library_without_view_sources(monkeypatch, tmp_path):
    """Those entry points are new symbols, not a reinterpreted field, so a library without them still loads and runs every
    other form; a call with a table names the missing probe."""
    old = [s for s in _lib.EXPORTS if s not in _lib.VIEW_SOURCES_EXPORTS]
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    lib = _lib.load()
    assert not hasattr(lib, "epi_fusion_view_sources")
    with pytest.raises(RuntimeError, match="epi_fusion_view_sources"):
        epi.epipolar_fusion_views(torch.zeros(2, 1, 8, 8, 8), torch.zeros(2, 1, 3, 4), K=8, sources=[[1], [0]])
    with pytest.raises(RuntimeError, match="no CPU implementation"):           # the all-others form goes on to its own checks
        epi.epipolar_fusion_views(torch.zeros(2, 1, 8, 8, 8), torch.zeros(2, 1, 3, 4), K=8)
