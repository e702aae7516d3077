"""CPU: the C-ABI library loads, exports every symbol include/epipolar_b200.h declares, its struct
mirror matches, and argument validation works without touching a GPU."""
import ctypes
import os
import re

import pytest

from epipolar_transformers_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(epi_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib):
    names = declared_functions()
    assert set(names) == set(_lib.EXPORTS)
    for n in names:
        assert hasattr(lib, n), n
    assert lib.epi_version() == _lib.EPI_ABI_VERSION


def test_struct_layout_matches_header():
    """field order/types of the ctypes mirror follow the header's struct, and the size agrees with a C compile."""
    import subprocess, tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "sz.c")
        open(c, "w").write('#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu", sizeof(EpiFusionParams),'
                           ' __builtin_offsetof(EpiFusionParams, N), __builtin_offsetof(EpiFusionParams, variant));return 0;}' % HEADER)
        exe = os.path.join(d, "sz")
        subprocess.check_call(["gcc", c, "-o", exe])
        size, off_n, off_var = map(int, subprocess.check_output([exe]).split())
    assert ctypes.sizeof(_lib.EpiFusionParams) == size
    assert _lib.EpiFusionParams.N.offset == off_n
    assert _lib.EpiFusionParams.variant.offset == off_var


def test_validation_without_gpu(lib):
    p = _lib.EpiFusionParams()
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1          # EPI_EINVAL: null tensors
    assert b"non-null" in lib.epi_last_error()
    buf = (ctypes.c_float * 4)()
    addr = ctypes.addressof(buf)
    p.feat_ref = addr; p.feat_src = addr; p.out = addr; p.P_ref = addr; p.P_src = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 1
    p.downsample = 4.0; p.img_scale = 1.0
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1          # K out of range
    assert b"SAMPLESIZE" in lib.epi_last_error()
    p.K = 8; p.C = 2000
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1
    assert lib.epi_fold_z_bn_f32(None, None, None, None, None, None, 1e-5, 8, None, None, None) == -1
    assert lib.epi_sample_locs_f32(None, None, None, 1, 8, 8, 8, 4.0, 1.0, 1e-3, 0, None) == -1


def test_workspace_plan(lib):
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = 4, 256, 64, 64, 64
    buf = (ctypes.c_float * 4)()
    p.feat_src = ctypes.addressof(buf)
    p.src_stride = (ctypes.c_int64 * 4)(256 * 4096, 4096, 64, 1)           # NCHW: needs staging
    p.out_stride = (ctypes.c_int64 * 4)(256 * 4096, 4096, 64, 1)           # NCHW output: pixel-major plane + transposition pass
    m = 4 * 256 * 64 * 64 * 4
    order = 4 * 4096 * 2                                                     # pixel order list (u16)
    geom = 256                                                               # 4 pairs x 44 B of pair constants, 256-B granules
    pipe = 2 * m + 256 + order + geom           # ref + src bf16 (hi, lo) planes, counter/error words, pixel order, pair constants
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == pipe + m      # + the pixel-major fp32 output plane
    p.out_stride = (ctypes.c_int64 * 4)(256 * 4096, 1, 64 * 256, 256)      # channels_last output: written directly
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == pipe
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) > 4 * 32 * 4 + geom + order + 512 * 4000   # keys + pair constants + order + work-item records
    p.cache = ctypes.addressof(buf)                                          # with a persistent cache they leave the workspace
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 2 * m + 256
    p.cache = None
    p.out_stride = (ctypes.c_int64 * 4)(256 * 4096, 4096, 64, 1)
    p.z_weight_folded = ctypes.addressof(buf)
    wpl = 256 * 256 * 4                                                      # folded z weight as bf16 (hi, lo) planes
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == pipe + m + wpl    # + pre-z bf16 planes + weight planes
    p.variant = _lib.EPI_VARIANT_SECTOR
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 3 * m + 256 + order
    assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) == 0
    p.variant = _lib.EPI_VARIANT_TILE
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 2 * m + 256   # 4x8 block tiles: no ref planes / order list
    p.variant = _lib.EPI_VARIANT_AUTO
    p.src_stride = (ctypes.c_int64 * 4)(256 * 4096, 1, 64 * 256, 256)      # channels_last
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == pipe + m + wpl    # tensor-core kernels stage bf16 (hi, lo) planes
    p.variant = _lib.EPI_VARIANT_WARP
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == m             # warp kernel reads channels_last in place


def test_kernel_selection_by_shape(lib):
    """Shape limits of the pipelined kernel as the ABI applies them (no GPU call): `epi_fusion_cache_bytes` is non-zero exactly
    when that kernel is selected (it is the only one that keeps cross-call state)."""
    def cache(C, H, W, K, variant=_lib.EPI_VARIANT_AUTO, N=2):
        p = _lib.EpiFusionParams()
        p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
        p.variant = variant
        return lib.epi_fusion_cache_bytes(ctypes.byref(p))
    assert cache(256, 64, 64, 64) > 0                       # BASELINE config 2
    assert cache(512, 64, 64, 128) > 0                      # wide: two query-panel halves; K = 128 fits because 4*max(H, W) = 256
    assert cache(520, 64, 64, 64) == 0                      # C > 512
    assert cache(260, 64, 64, 64) == 0                      # C % 8 != 0
    assert cache(64, 256, 256, 32) > 0                      # 65536 pixels: row-windowed union bitmap
    assert cache(64, 100, 400, 48) > 0                      # non-square above 16384 pixels
    assert cache(64, 300, 100, 16) == 0                     # more than 256 rows
    assert cache(64, 128, 128, 128) == 0                    # a single pixel's union (min(4K, 4*max)) exceeds 256 rows
    # automatic selection leaves K > 48 on maps of 2K+ pixels a side to the other kernels; forcing the kernel still works
    assert cache(256, 128, 128, 64) == 0 and cache(256, 256, 256, 64) == 0
    assert cache(256, 128, 128, 64, _lib.EPI_VARIANT_PIPE) > 0 and cache(256, 96, 96, 64) > 0 and cache(256, 256, 256, 48) > 0
    # workspace of the wide / large-map plans: operand planes + counters (+ order, pair constants without a cache)
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = 1, 512, 32, 32, 64
    p.out_stride = (ctypes.c_int64 * 4)(512 * 1024, 1, 32 * 512, 512)       # channels_last output
    m = 512 * 1024 * 4
    assert lib.epi_fusion_workspace_bytes(ctypes.byref(p)) == 2 * m + 256 + 1024 * 2 + 256


def test_plan_sizes_match_golden(lib):
    """Forward workspace, cache and backward workspace bytes over a sweep of every variant, dtype, epilogue, cache, n_src and
    layout on shapes on both sides of each kernel's limits, plus invalid params, equal the table recorded by
    oracle/make_golden_plan.py.  A planning change that moves a region shows up here."""
    import numpy as np
    from oracle import make_golden_plan as g
    want = np.load(g.GOLDEN)["sizes"]
    got = g.sizes(lib)
    assert got.shape == want.shape
    bad = np.flatnonzero((got != want).any(axis=1))
    cases = g.rows() + list(g.INVALID)
    assert bad.size == 0, "%d rows differ, first: %s got %s want %s" % (bad.size, cases[bad[0]], got[bad[0]], want[bad[0]])


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU/PyTorch fallback"):
        _lib.load()
