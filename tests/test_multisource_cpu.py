"""CPU: the several-sources-per-reference interface (EpiFusionParams.n_src, epi_find_peaks_best_f32) and its Python entry
points, checked without a GPU: struct layout, workspace and cache sizes, argument validation."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_n_src_offset_matches_header_and_size_is_unchanged():
    """n_src is carved out of the first remaining reserved word, right after feat_dtype; the struct keeps its size and every
    other field its offset (compared with the layout before the field existed)."""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "off.c")
        open(c, "w").write(
            '#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%d", __builtin_offsetof(EpiFusionParams, n_src),'
            ' __builtin_offsetof(EpiFusionParams, reserved), sizeof(EpiFusionParams), EPI_ABI_VERSION);return 0;}' % HEADER)
        exe = os.path.join(d, "off")
        subprocess.check_call(["gcc", c, "-o", exe])
        off, res, size, ver = map(int, subprocess.check_output([exe]).split())
    P = _lib.EpiFusionParams
    assert P.n_src.offset == off == P.feat_dtype.offset + 4
    assert P.reserved.offset == res == off + 4
    assert ctypes.sizeof(P) == size and ver == _lib.EPI_ABI_VERSION == 3

    class Before(ctypes.Structure):             # the v3 layout with reserved[2] after feat_dtype
        _fields_ = [f for f in P._fields_ if f[0] not in ("n_src", "reserved")]
        _fields_.insert([f[0] for f in _fields_].index("feat_dtype") + 1, ("reserved", ctypes.c_int32 * 2))
    assert ctypes.sizeof(Before) == size
    for name, _ in P._fields_:
        if name not in ("n_src", "reserved"):
            assert getattr(P, name).offset == getattr(Before, name).offset, name
    assert Before.reserved.offset == P.n_src.offset


def _cfg2(p, feat_dtype=_lib.EPI_DTYPE_F32):
    """the cfg2 pipelined shape: N=4, C=256, 64x64, K=64, NCHW out"""
    p.N, p.C, p.H, p.W, p.K = 4, 256, 64, 64, 64
    p.out_stride = (ctypes.c_int64 * 4)(256 * 4096, 4096, 64, 1)
    p.feat_dtype = feat_dtype
    return p


M = 4 * 256 * 64 * 64 * 4          # bytes of one fp32 copy of the N = 4 reference maps


@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16], ids=["f32", "bf16"])
def test_workspace_counts_reference_planes_once(lib, dtype):
    """n_src = 0 and 1 size exactly what one source sizes.  With n_src = 3 the workspace grows by the planes of two more source
    maps and two more pre-z maps only: the reference planes are staged once, not three times (staging them per source would
    add another 2 x (one fp32 map) for fp32 / fp16 maps)."""
    sizes = {}
    for n_src in (0, 1, 3):
        p = _cfg2(_lib.EpiFusionParams(), dtype)
        p.z_weight_folded = 256; p.z_bias_folded = 256          # the z GEMM path (sizes only: nothing is dereferenced)
        p.cache = 256                                           # a persistent cache holds the per-pair records
        p.n_src = n_src
        sizes[n_src] = lib.epi_fusion_workspace_bytes(ctypes.byref(p))
    assert sizes[0] == sizes[1] > 0
    planes_per_src_map = M if dtype == _lib.EPI_DTYPE_F32 else M // 2      # bf16 maps: hi planes only
    assert sizes[3] - sizes[1] == 2 * planes_per_src_map + 2 * M, sizes


def test_workspace_without_cache_covers_pair_records(lib):
    """without a persistent cache the workspace also holds the pixel order and pair constants, per pair"""
    p = _cfg2(_lib.EpiFusionParams())
    base = lib.epi_fusion_workspace_bytes(ctypes.byref(p))
    p.n_src = 3
    three = lib.epi_fusion_workspace_bytes(ctypes.byref(p))
    order1, order3 = 4 * 4096 * 2, 12 * 4096 * 2                          # uint16 per pixel and pair (multiples of 256)
    geom1, geom3 = 256, 768                                               # 44-byte PairGeom per pair, 256-byte aligned
    # fp32 maps, NCHW out: + 2 source maps of (hi, lo) planes + 2 pixel-major output maps + the per-pair records
    assert three - base == 2 * M + 2 * M + (order3 - order1) + (geom3 - geom1)


def test_cache_covers_s_times_n_pairs(lib):
    p = _cfg2(_lib.EpiFusionParams())
    one = lib.epi_fusion_cache_bytes(ctypes.byref(p))
    p.n_src = 1
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == one > 0
    p.n_src = 3
    three = lib.epi_fusion_cache_bytes(ctypes.byref(p))
    q = _cfg2(_lib.EpiFusionParams())
    q.N = 12                                                              # the cache is per pair: S·N = 12 pairs ...
    twelve = lib.epi_fusion_cache_bytes(ctypes.byref(q))
    # ... plus, per further source, the half-tile work records a single-source call keeps
    assert twelve < three < 2 * twelve, (one, three, twelve)


def _params_on_host_buffer():
    buf = (ctypes.c_float * 4)()
    addr = ctypes.addressof(buf)
    p = _lib.EpiFusionParams()
    p.feat_ref = addr; p.feat_src = addr; p.out = addr; p.P_ref = addr; p.P_src = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 8
    p.downsample = 4.0; p.img_scale = 1.0
    return p, buf


def test_abi_rejects_negative_n_src(lib):
    p, _buf = _params_on_host_buffer()
    p.n_src = -1
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1        # EPI_EINVAL, before any CUDA call
    assert b"n_src" in lib.epi_last_error()
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 0
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == 0


def test_abi_rejects_pairs_beyond_grid_limit(lib):
    p, _buf = _params_on_host_buffer()
    p.N, p.n_src = 40000, 2
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1
    assert b"65535" in lib.epi_last_error()


def test_abi_rejects_bad_best_peak_arguments(lib):
    buf = (ctypes.c_float * 4)()
    a = ctypes.addressof(buf)
    assert lib.epi_find_peaks_best_f32(a, a, a, None, 0, 1, 1, 8, 8, 1.0, 4.0, 1e-6, 0, None) == -1
    assert lib.epi_find_peaks_best_f32(None, a, a, None, 2, 1, 1, 8, 8, 1.0, 4.0, 1e-6, 0, None) == -1
    assert lib.epi_find_peaks_best_f32(a, a, a, None, 2, 1, 1, 8, 8, 0.2, 4.0, 1e-6, 0, None) == -1


def _multi(ref, srcs, P1=None, P2=None, **kw):
    N = ref.shape[0]
    S = len(srcs) if isinstance(srcs, (list, tuple)) else srcs.shape[0]
    P1 = torch.zeros(N, 3, 4) if P1 is None else P1
    P2 = torch.zeros(S, N, 3, 4) if P2 is None else P2
    return epi.epipolar_fusion_multi(ref, srcs, P1, P2, K=8, **kw)


def test_python_shape_and_dtype_errors():
    x = torch.zeros(2, 8, 8, 8)
    srcs = torch.zeros(3, 2, 8, 8, 8)
    with pytest.raises(ValueError, match="feat_srcs"):
        _multi(x, x)                                                      # 4-D: not [S,N,C,H,W]
    with pytest.raises(ValueError, match="feat_srcs"):
        _multi(x, [])
    with pytest.raises(ValueError, match="share shape"):
        _multi(x, [x, torch.zeros(2, 8, 8, 4)])
    with pytest.raises(ValueError, match="feat_ref's shape"):
        _multi(x, torch.zeros(3, 1, 8, 8, 8))
    with pytest.raises(ValueError, match=r"P_srcs must be \[S,N,3,4\]"):
        _multi(x, srcs, P2=torch.zeros(2, 3, 4))
    with pytest.raises(ValueError, match=r"sample_locs_in must be \[K,S,N,H,W,2\]"):
        _multi(x, srcs, sample_locs_in=torch.zeros(8, 6, 8, 8, 2))
    with pytest.raises(ValueError, match="out must be"):
        _multi(x, srcs, out=torch.zeros(6, 8, 8, 8))
    with pytest.raises(TypeError, match="same dtype"):
        _multi(x, srcs.bfloat16())
    with pytest.raises(TypeError, match="float32, bfloat16 or float16"):
        _multi(x.double(), srcs.double())
    with pytest.raises(TypeError, match="out must be float32"):
        _multi(x, srcs, out=torch.zeros(3, 2, 8, 8, 8, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="no CPU implementation"):     # valid arguments on the CPU are still refused
        _multi(x, [x, x, x])


def test_peak_best_argument_errors():
    with pytest.raises(ValueError, match=r"\[S,B,J,H,W\]"):
        epi.find_tensor_peak_best(torch.zeros(2, 3, 8, 8), 1.0, 4.0)
    with pytest.raises(ValueError, match="divide zero"):
        epi.find_tensor_peak_best(torch.zeros(2, 1, 3, 1, 8), 1.0, 4.0)
    with pytest.raises(ValueError, match="radius"):
        epi.find_tensor_peak_best(torch.zeros(2, 1, 3, 8, 8), 0.0, 4.0)
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        epi.find_tensor_peak_best(torch.zeros(2, 1, 3, 8, 8), 1.0, 4.0)


def test_forward_multi_refuses_training_mode_with_z():
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(8, 8), NFEATS=8), EPIPOLAR=dict(SAMPLESIZE=8, PARAMETERIZED=("z",)))
    m = epi.Epipolar(cfg=cfg).train()
    x = torch.zeros(2, 8, 8, 8)
    with pytest.raises(RuntimeError, match="eval mode"):
        m.forward_multi(x, torch.zeros(3, 2, 8, 8, 8), torch.zeros(2, 3, 4), torch.zeros(3, 2, 3, 4))
