"""CPU: the ABI of the deterministic backward (EpiFusionBwdParams.deterministic): the field's place in the struct, the exact
workspace it adds, its validation, the Python argument check, and load() refusing a library that predates the field."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from epipolar_transformers_b200 import _lib, build
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_field_offset_and_struct_size_match_c():
    """`deterministic` takes reserved[0]'s place: the struct keeps its size and every other offset."""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "off.c")
        open(c, "w").write('#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu", sizeof(EpiFusionBwdParams),'
                           ' __builtin_offsetof(EpiFusionBwdParams, feat_dtype), __builtin_offsetof(EpiFusionBwdParams, deterministic),'
                           ' __builtin_offsetof(EpiFusionBwdParams, reserved));return 0;}' % HEADER)
        exe = os.path.join(d, "off")
        subprocess.check_call(["gcc", c, "-o", exe])
        size, off_dt, off_det, off_res = map(int, subprocess.check_output([exe]).split())
    B = _lib.EpiFusionBwdParams
    assert ctypes.sizeof(B) == size
    assert (B.feat_dtype.offset, B.deterministic.offset, B.reserved.offset) == (off_dt, off_det, off_res)
    assert off_det == off_dt + 4 and off_res == off_det + 4
    assert B.reserved.size == 8
    # size and feat_dtype offset of the layout before the field existed (feat_dtype, int32 reserved[3]; LP64)
    assert (size, off_dt) == (328, 308)


def _bwd_params(N, C, H, W, K, dtype=_lib.EPI_DTYPE_F32, det=0):
    p = _lib.EpiFusionBwdParams()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.feat_dtype = dtype
    p.deterministic = det
    return p


def _align(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("shape", [(4, 256, 64, 64, 64), (3, 17, 12, 20, 33), (1, 4, 2, 2, 2)])
@pytest.mark.parametrize("dtype", [_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16])
def test_deterministic_workspace_bytes(lib, shape, dtype):
    """deterministic = 1 appends an int64 accumulator (8·N·H·W·C bytes), one 32-bit word per pair and the [N,K,H·W] float2
    coefficients, each region 256-byte aligned, behind the default path's regions, which are unchanged."""
    N, C, H, W, K = shape
    base = lib.epi_fusion_backward_workspace_bytes(ctypes.byref(_bwd_params(N, C, H, W, K, dtype, 0)))
    fmap = N * C * H * W * 4
    assert base == _align(fmap) * (2 if dtype == _lib.EPI_DTYPE_F32 else 4)
    det = lib.epi_fusion_backward_workspace_bytes(ctypes.byref(_bwd_params(N, C, H, W, K, dtype, 1)))
    assert det == base + _align(8 * N * H * W * C) + _align(4 * N) + _align(8 * N * K * H * W)


def test_deterministic_value_2_is_einval(lib):
    p = _bwd_params(2, 8, 4, 4, 4, det=2)
    for name in ("feat_ref", "feat_src", "P_ref", "P_src", "attn", "grad_out", "grad_src", "workspace"):
        setattr(p, name, 256)                      # non-null dummies: validation rejects the call before touching memory
    assert lib.epi_fusion_backward_f32(ctypes.byref(p), None) == -1
    assert lib.epi_last_error() == b"deterministic must be 0 or 1"
    assert lib.epi_fusion_backward_deterministic() == 1


@pytest.mark.parametrize("bad", [1, 0, "yes", 1.0])
def test_python_deterministic_must_be_bool(bad):
    f = torch.zeros(1, 4, 4, 4)
    with pytest.raises(TypeError, match="deterministic must be None or a bool"):
        epipolar_fusion_backward(f, f, None, None, torch.zeros(1, 2, 4, 4), f, K=2, deterministic=bad)


def test_load_refuses_library_without_deterministic_export(monkeypatch, tmp_path):
    """A library built before the field would read `deterministic` as a reserved word and ignore it: load() refuses it."""
    old = [s for s in _lib.EXPORTS if s != "epi_fusion_backward_deterministic"]
    assert len(old) == len(_lib.EXPORTS) - 1
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    with pytest.raises(RuntimeError, match="epi_fusion_backward_deterministic"):
        _lib.load()
