"""CPU: the views form of the forward (EpiFusionParams.n_views: every view of a frame against every other view in one call) and
its Python entry points, checked without a GPU: struct layout, argument refusals, workspace and cache sizes, Python errors."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")
EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_n_views_takes_the_last_reserved_word():
    """n_views shares reserved[0]'s storage: same offset in C and in the ctypes mirror, and the struct keeps its size"""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "off.c")
        open(c, "w").write(
            '#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu", __builtin_offsetof(EpiFusionParams, n_views),'
            ' __builtin_offsetof(EpiFusionParams, reserved), sizeof(EpiFusionParams));return 0;}' % HEADER)
        exe = os.path.join(d, "off")
        subprocess.check_call(["gcc", c, "-o", exe])
        off, res, size = map(int, subprocess.check_output([exe]).split())
    P = _lib.EpiFusionParams
    assert off == res == P.reserved.offset == P.n_src.offset + 4 and ctypes.sizeof(P) == size
    p = P()
    p.n_views = 4
    assert p.reserved[0] == 4 and p.n_views == 4


# ---- ABI refusals (EPI_EINVAL before any CUDA call) ------------------------------------------------------------------------
def _views_params(V=3):
    buf = (ctypes.c_float * 64)()
    addr = ctypes.addressof(buf)
    p = _lib.EpiFusionParams()
    p.feat_ref = addr; p.out = addr; p.P_ref = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 8
    p.downsample = 4.0; p.img_scale = 1.0
    p.n_views = V
    return p, buf


@pytest.mark.parametrize("case", ["n_views_1", "n_views_negative", "feat_src", "P_src", "n_src_2", "locs_misaligned",
                                  "too_many_pairs"])
def test_abi_refusals(lib, case):
    p, buf = _views_params()
    addr = ctypes.addressof(buf)
    if case == "n_views_1":
        p.n_views = 1
    elif case == "n_views_negative":
        p.n_views = -2
    elif case == "feat_src":
        p.feat_src = addr
    elif case == "P_src":
        p.P_src = addr
    elif case == "n_src_2":
        p.n_src = 2
    elif case == "locs_misaligned":
        p.sample_locs_in = addr + 4                              # (x, y) pairs are read as one 8-byte vector
    else:
        p.N, p.n_views = 2000, 7                                 # 7·6·2000 pairs > 65535
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == EINVAL
    msg = lib.epi_last_error()
    assert {"n_views_1": b"n_views", "n_views_negative": b"n_views", "feat_src": b"must be null", "P_src": b"must be null",
            "n_src_2": b"n_src", "locs_misaligned": b"8-byte", "too_many_pairs": b"65535"}[case] in msg, msg


def test_size_queries_answer_zero_for_unplannable_views(lib):
    for kw in ({"n_views": 1}, {"n_views": -1}, {"n_views": 3, "n_src": 2}, {"n_views": 300}):
        p, _buf = _views_params()
        for k, v in kw.items():
            setattr(p, k, v)
        assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 0, kw
        assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == 0, kw
    assert lib.epi_fusion_views() == 1


# ---- workspace and cache sizes -------------------------------------------------------------------------------------------
C, H, W, K = 256, 64, 64, 64                                     # the cfg2 shape (pipelined kernel, 64-pixel items)
PX = H * W
MAP1 = C * PX * 4                                                # one fp32 map of one item
REC_BYTES = 4352                                                 # the pipelined kernel's plan-cache record slot


def al(b):
    return (b + 255) // 256 * 256


def pipe_workspace(V, N, lo, z, cache):
    """[view planes (hi, + lo)] [fused feature: bf16 (hi, lo) for the z GEMM, else the fp32 pixel-major plane] [counters]
    [z weight planes] [pixel order + pair constants unless cached].  The V·N view items are staged once: no source planes."""
    NR, NP = V * N, V * (V - 1) * N
    b = al(NR * MAP1 if lo else NR * MAP1 // 2) + NP * MAP1 + 256
    if z:
        b += 2 * C * C * 2
    if not cache:
        b += al(NP * PX * 2) + al(NP * 44)
    return b


def pipe_cache(V, N):
    """[keys: 32 words per pair] [pair constants] [pixel order] [work records: whole 32-pixel slots + per view pair the
    half-item slots a one-source call on N items keeps]"""
    NP = V * (V - 1) * N
    records = NP * ((PX + 31) // 32) + V * (V - 1) * (256 + N)
    return al(NP * 128) + al(NP * 44) + al(NP * PX * 2) + al(records * REC_BYTES)


def _cfg2(V, N, dtype=_lib.EPI_DTYPE_F32, z=True, cache=True):
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.ref_stride = (ctypes.c_int64 * 4)(C * PX, PX, W, 1)
    p.out_stride = (ctypes.c_int64 * 4)(C * PX, PX, W, 1)
    p.feat_dtype = dtype
    p.n_views = V
    if z:
        p.z_weight_folded = p.z_bias_folded = 256                # sizes only: nothing is dereferenced
    if cache:
        p.cache = 256
    return p


@pytest.mark.parametrize("V,N", [(2, 1), (4, 1), (4, 4), (5, 2)])
@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16, _lib.EPI_DTYPE_F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("z", [True, False], ids=["z", "noz"])
@pytest.mark.parametrize("cache", [True, False], ids=["cache", "nocache"])
def test_pipe_sizes_match_formula(lib, V, N, dtype, z, cache):
    p = _cfg2(V, N, dtype, z, cache)
    lo = dtype != _lib.EPI_DTYPE_BF16                            # bf16 maps have no lo planes
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == pipe_workspace(V, N, lo, z, cache)
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == pipe_cache(V, N)


def test_views_cache_equals_multi_source_cache(lib):
    """per pair, the views form keeps exactly the records a multi-source call with V·(V−1) sources keeps"""
    p = _cfg2(4, 2)
    q = _cfg2(0, 2)
    q.n_src = 12
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == lib.epi_fusion_cache_bytes(ctypes.byref(q))


@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16], ids=["f32", "bf16"])
def test_warp_sizes_stage_each_view_once(lib, dtype):
    """warp kernel, NCHW maps: fp32 maps get one channels-last copy of the V·N views (the source of every pair); a bf16 map's
    fp32 copy (the query) is that source already, so nothing else is staged"""
    V, N, c, h, w = 3, 2, 64, 32, 32
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = N, c, h, w, 16
    p.ref_stride = (ctypes.c_int64 * 4)(c * h * w, h * w, w, 1)
    p.out_stride = (ctypes.c_int64 * 4)(c * h * w, h * w, w, 1)
    p.variant, p.feat_dtype, p.n_views = _lib.EPI_VARIANT_WARP, dtype, V
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == al(V * N * c * h * w * 4)


def test_n_views_zero_keeps_todays_sizes(lib):
    """n_views = 0 written explicitly sizes every shape of the plan-size table exactly as recorded before the field existed"""
    from oracle import make_golden_plan as g
    want = np.load(g.GOLDEN)["sizes"]
    for i, row in enumerate(g.rows()):
        p, _ = g._params(row, n_views=0)
        got = (lib.epi_fusion_workspace_bytes(ctypes.byref(p)), lib.epi_fusion_cache_bytes(ctypes.byref(p)))
        assert got == tuple(int(x) for x in want[i, :2]), row


# ---- the Python entry points -----------------------------------------------------------------------------------------------
def _views(feats, P=None, **kw):
    V, N = (len(feats), feats[0].shape[0]) if isinstance(feats, (list, tuple)) else tuple(feats.shape[:2])
    P = torch.zeros(V, N, 3, 4) if P is None else P
    return epi.epipolar_fusion_views(feats, P, K=8, **kw)


def test_python_argument_errors():
    f = torch.zeros(3, 2, 8, 8, 8)
    with pytest.raises(ValueError, match=r"\[V,N,C,H,W\]"):
        _views(torch.zeros(2, 8, 8, 8), P=torch.zeros(2, 1, 3, 4))
    with pytest.raises(ValueError, match="at least two views"):
        _views(f[:1])
    with pytest.raises(ValueError, match="at least two views"):
        _views([f[0]])
    with pytest.raises(ValueError, match="share shape"):
        _views([f[0], torch.zeros(2, 8, 8, 4)])
    with pytest.raises(ValueError, match=r"P must be \[V,N,3,4\]"):
        _views(f, P=torch.zeros(2, 2, 3, 4))
    with pytest.raises(ValueError, match=r"sample_locs_in must be \[K,V,V-1,N,H,W,2\]"):
        _views(f, sample_locs_in=torch.zeros(8, 3, 3, 2, 8, 8, 2))
    with pytest.raises(ValueError, match="out must be"):
        _views(f, out=torch.zeros(3, 3, 2, 8, 8, 8))
    with pytest.raises(TypeError, match="float32, bfloat16 or float16"):
        _views(f.double())
    with pytest.raises(TypeError, match="out must be float32"):
        _views(f, out=torch.zeros(3, 2, 2, 8, 8, 8, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="no CPU implementation"):   # valid arguments on the CPU are still refused
        _views(list(f))


def test_forward_views_refuses_training_mode_with_z():
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(8, 8), NFEATS=8), EPIPOLAR=dict(SAMPLESIZE=8, PARAMETERIZED=("z",)))
    m = epi.Epipolar(cfg=cfg).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        m.forward_views(torch.zeros(3, 2, 8, 8, 8), torch.zeros(3, 2, 3, 4))


def test_load_refuses_library_without_views_export(monkeypatch, tmp_path):
    """A library built before n_views would read it as a reserved word and run a one-source call: load() refuses it."""
    old = [s for s in _lib.EXPORTS if s != "epi_fusion_views"]
    assert len(old) == len(_lib.EXPORTS) - 1
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    with pytest.raises(RuntimeError, match="epi_fusion_views"):
        _lib.load()
    with pytest.raises(RuntimeError, match="epi_fusion_views"):
        epi.epipolar_fusion_views(torch.zeros(2, 1, 8, 8, 8), torch.zeros(2, 1, 3, 4), K=8)
