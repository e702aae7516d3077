"""CPU: the backward of the views form (epi_fusion_views_backward_*) and its Python entry points, checked without a GPU: every
ABI refusal with its message, the workspace size against a formula, the Python errors, and loading a library built before the
entry points."""
import ctypes
import subprocess

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build

EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def tbl(rows):
    t = np.ascontiguousarray(rows, dtype=np.int32)
    return t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), t.shape[1], t        # keep `t` alive with the pointer


def al(v):
    return (v + 255) // 256 * 256


def bwd_params(N=2, C=8, H=4, W=4, K=4, dtype=_lib.EPI_DTYPE_F32, det=0):
    """a valid views backward of 3 views over non-null dummy pointers: every refusal below fires before memory is touched"""
    p = _lib.EpiFusionBwdParams()
    for name in ("feat_ref", "P_ref", "attn", "grad_out", "grad_ref", "workspace"):
        setattr(p, name, 256)
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.downsample, p.img_scale, p.eps, p.softmax_scale = 4.0, 1.0, 1e-3, 0.125
    p.grad_keys = p.grad_vals = 1
    p.feat_dtype = dtype
    p.deterministic = det
    return p


# ---- ABI refusals (EPI_EINVAL before any CUDA call) ------------------------------------------------------------------------
# case -> (change, message): table refusals as in the source-table forward, the views-form refusals and those of the one-pair
# backward
REFUSALS = {
    "null_params": ("null_params", b"params is null"),
    "n_views_1": ("n_views_1", b"n_views must be >= 2"),
    "null_table": ("null_table", b"sources_host is null"),
    "s_zero": ("s_zero", b"S (sources per view) must be >= 1"),
    "entry_negative": ([[1], [-1], [0]], b"is not a view in [0, 3)"),
    "entry_too_large": ([[1], [3], [0]], b"is not a view in [0, 3)"),
    "self_pair": ([[1], [1], [0]], b"with itself"),
    "too_many_entries": ("entries", b"EPI_VIEW_SOURCES_MAX"),
    "too_many_pairs": ("pairs", b"65535"),
    "all_others_too_many_pairs": ("all_others_pairs", b"65535"),
    "feat_src": ("feat_src", b"feat_src, P_src and grad_src must be null"),
    "P_src": ("P_src", b"feat_src, P_src and grad_src must be null"),
    "grad_src": ("grad_src", b"feat_src, P_src and grad_src must be null"),
    "null_attn": ("attn", b"must be non-null"),
    "no_cameras": ("P_ref", b"P_ref/P_src required without sample_locs_in"),
    "k1": ("k1", b"bad shape"),
    "h1": ("h1", b"bad shape"),
    "c513": ("c513", b"backward supports C <= 128, or C <= 512 with C % 4 == 0"),
    "c130": ("c130", b"backward supports C <= 128, or C <= 512 with C % 4 == 0"),
    "dtype": ("dtype", b"unknown feat_dtype"),
    "deterministic_2": ("det2", b"deterministic must be 0 or 1"),
    "locs_misaligned": ("locs", b"8-byte aligned"),
}


def _refused(case):
    p = bwd_params()
    V = 3
    ptr, S, t = tbl([[1], [2], [0]])
    change = REFUSALS[case][0]
    if isinstance(change, list):
        ptr, S, t = tbl(change)
    elif change == "null_params":
        p = None
    elif change == "n_views_1":
        V = 1
    elif change == "null_table":
        ptr = None
    elif change == "s_zero":
        S = 0
    elif change == "entries":                                    # 17 views · 16 sources = 272 > 256 entries
        V = 17
        ptr, S, t = tbl([[(v + 1 + j) % 17 for j in range(16)] for v in range(17)])
    elif change == "pairs":                                      # 3·2·11000 pairs > 65535
        p.N = 11000
        ptr, S, t = tbl([[1, 2], [2, 0], [0, 1]])
    elif change == "all_others_pairs":                           # 30·29·76 pairs > 65535
        V, ptr, S, p.N = 30, None, 0, 76
    elif change in ("feat_src", "P_src", "grad_src"):
        setattr(p, change, 256)
    elif change in ("attn", "P_ref"):
        setattr(p, change, None)
    elif change == "k1":
        p.K = 1
    elif change == "h1":
        p.H = 1
    elif change == "c513":
        p.C = 513
    elif change == "c130":
        p.C = 130
    elif change == "dtype":
        p.feat_dtype = 3
    elif change == "det2":
        p.deterministic = 2
    elif change == "locs":
        p.sample_locs_in = 260
    return p, V, ptr, S, t


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_abi_refusals(lib, case):
    p, V, ptr, S, _t = _refused(case)
    assert lib.epi_fusion_views_backward_f32(None if p is None else ctypes.byref(p), V, ptr, S, None) == EINVAL
    msg = lib.epi_last_error()
    assert REFUSALS[case][1] in msg, msg


@pytest.mark.parametrize("case", ["null_params", "n_views_1", "null_table", "s_zero", "entry_negative", "self_pair",
                                  "too_many_entries", "too_many_pairs", "all_others_too_many_pairs"])
def test_workspace_query_answers_zero_for_unplannable_calls(lib, case):
    p, V, ptr, S, _t = _refused(case)
    assert lib.epi_fusion_views_backward_workspace_bytes(None if p is None else ctypes.byref(p), V, ptr, S) == 0


def test_probe(lib):
    assert lib.epi_fusion_views_backward() == 1


# ---- workspace: the V·N view maps staged once, per-item sums, one query term per pair (+ the fixed-point state) -------------
def views_workspace(V, S, N, C, H, W, K, det):
    NI, NP, item = V * N, V * S * N, C * H * W * 4
    b = 2 * al(NI * item) + al(NP * item)
    if det:
        b += al(2 * NI * item) + al(4 * NI) + al(8 * NP * H * W * K)
    return b


@pytest.mark.parametrize("det", [0, 1], ids=["default", "det"])
@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16, _lib.EPI_DTYPE_F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("V,rows,N,C,H,W,K", [
    (4, [[1], [2], [3], [0]], 4, 256, 64, 64, 64),               # the training shape: nearest camera, 16 pairs
    (3, [[1, 2], [2, 0], [0, 0]], 2, 17, 13, 17, 33),            # duplicates, an odd map and C
    (5, None, 1, 64, 12, 16, 2),                                 # every other view
])
def test_workspace_matches_formula(lib, V, rows, N, C, H, W, K, dtype, det):
    p = bwd_params(N, C, H, W, K, dtype, det)
    if rows is None:
        ptr, S, t = None, 0, None
        Sw = V - 1
    else:
        ptr, S, t = tbl(rows)
        Sw = S
    assert lib.epi_fusion_views_backward_workspace_bytes(ctypes.byref(p), V, ptr, S) == views_workspace(V, Sw, N, C, H, W, K, det)


def test_all_others_table_needs_the_same_workspace(lib):
    p = bwd_params(2, 64, 12, 16, 8, det=1)
    ptr, S, _t = tbl([[j + (j >= v) for j in range(3)] for v in range(4)])
    assert lib.epi_fusion_views_backward_workspace_bytes(ctypes.byref(p), 4, ptr, S) == \
        lib.epi_fusion_views_backward_workspace_bytes(ctypes.byref(p), 4, None, 0)


# ---- the Python entry points -----------------------------------------------------------------------------------------------
def _bwd(feats, P=None, sources=None, **kw):
    V, N, C, H, W = feats.shape
    S = V - 1 if sources is None else len(sources[0])
    kw.setdefault("attn", torch.zeros(V, S, N, 4, H, W))
    kw.setdefault("grad_out", torch.zeros(V, S, N, C, H, W))
    return epi.epipolar_fusion_views_backward(feats, torch.zeros(V, N, 3, 4) if P is None else P, K=4, sources=sources, **kw)


def test_python_refusals(lib):
    f = torch.zeros(3, 2, 8, 6, 6)
    with pytest.raises(ValueError, match=r"\[V,N,C,H,W\]"):
        epi.epipolar_fusion_views_backward(f[0], None, None, None, K=4)
    with pytest.raises(ValueError, match="at least two views"):
        _bwd(f[:1])
    with pytest.raises(ValueError, match=r"attn must be a \[V,S,N,K,H,W\]"):
        _bwd(f, sources=[[1], [2], [0]], attn=torch.zeros(3, 2, 2, 4, 6, 6))
    with pytest.raises(ValueError, match=r"grad_out must be a \[V,V-1,N,C,H,W\]"):
        _bwd(f, grad_out=torch.zeros(3, 1, 2, 8, 6, 6))
    with pytest.raises(ValueError, match=r"grad_attn must be a \[V,S,N,K,H,W\]"):
        _bwd(f, sources=[[1], [2], [0]], grad_attn=torch.zeros(3, 1, 2, 5, 6, 6))
    with pytest.raises(ValueError, match="itself"):
        _bwd(f, sources=[[1], [1], [0]])
    with pytest.raises(TypeError, match="float32, bfloat16 or float16"):
        _bwd(f.double())
    with pytest.raises(TypeError, match="deterministic must be None or a bool"):
        _bwd(f, deterministic=1)
    with pytest.raises(RuntimeError, match="no CPU implementation"):   # valid arguments on the CPU are still refused
        _bwd(f, sources=torch.tensor([[1], [2], [0]]))


def test_dtype_mismatch_between_views_refused(lib):
    with pytest.raises(ValueError, match="sharing shape, dtype and device"):
        epi.epipolar_fusion_views_backward([torch.zeros(2, 8, 6, 6), torch.zeros(2, 8, 6, 6, dtype=torch.float16)], None, None,
                                           None, K=4)


def test_cuda_table_refused_without_gpu(monkeypatch, lib):
    """a table that says it lives on the GPU is refused before anything reads it"""
    t = torch.tensor([[1], [0]])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(TypeError, match="synchronise"):
        _bwd(torch.zeros(2, 1, 8, 6, 6), sources=t)


def test_forward_views_train_accepts_training_mode_with_z():
    """unlike forward_views, the differentiable form runs in training mode (z and BatchNorm stay PyTorch's): on CPU maps it gets
    as far as the device check"""
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(8, 8), NFEATS=8), EPIPOLAR=dict(SAMPLESIZE=8, PARAMETERIZED=("z",)))
    m = epi.Epipolar(cfg=cfg).train()
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        m.forward_views_train(torch.zeros(3, 2, 8, 8, 8, requires_grad=True), torch.zeros(3, 2, 3, 4), sources=[[1], [2], [0]])


# ---- a library built before the views backward ----------------------------------------------------------------------------
def test_load_accepts_library_without_views_backward(monkeypatch, tmp_path):
    """The views backward is three new symbols, not a reinterpreted field, so a library without them still loads and runs every
    other form; a views-backward call names the missing probe."""
    old = [s for s in _lib.EXPORTS if s not in _lib.VIEWS_BACKWARD_EXPORTS]
    assert len(old) == len(_lib.EXPORTS) - 3
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 1) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    lib = _lib.load()
    assert not hasattr(lib, "epi_fusion_views_backward")
    with pytest.raises(RuntimeError, match="epi_fusion_views_backward"):
        _bwd(torch.zeros(2, 1, 8, 6, 6), sources=[[1], [0]])
    with pytest.raises(RuntimeError, match="no CPU implementation"):           # the views forward goes on to its own checks
        epi.epipolar_fusion_views(torch.zeros(2, 1, 8, 8, 8), torch.zeros(2, 1, 3, 4), K=8, sources=[[1], [0]])
