"""CPU: the bfloat16 / float16 feature-map interface of the C ABI and of the Python entry points, checked without a GPU
(the library loads without a device; argument validation happens before any CUDA call)."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epipolar_b200.h")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_feat_dtype_offsets_match_header():
    """feat_dtype is carved out of the first reserved word: its offset agrees with a C compile, and the struct sizes and the
    offsets of the surrounding fields did not move."""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "off.c")
        open(c, "w").write(
            '#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu %%d %%d %%d %%d",'
            ' __builtin_offsetof(EpiFusionParams, feat_dtype), __builtin_offsetof(EpiFusionParams, reserved),'
            ' sizeof(EpiFusionParams), __builtin_offsetof(EpiFusionBwdParams, feat_dtype), __builtin_offsetof(EpiFusionBwdParams, reserved),'
            ' sizeof(EpiFusionBwdParams), EPI_ABI_VERSION, EPI_DTYPE_F32, EPI_DTYPE_BF16, EPI_DTYPE_F16);return 0;}' % HEADER)
        exe = os.path.join(d, "off")
        subprocess.check_call(["gcc", c, "-o", exe])
        vals = list(map(int, subprocess.check_output([exe]).split()))
    f_off, f_res, f_size, b_off, b_res, b_size, ver, d32, dbf, dh = vals
    assert _lib.EpiFusionParams.feat_dtype.offset == f_off == _lib.EpiFusionParams.variant.offset + 4
    assert _lib.EpiFusionParams.reserved.offset == f_res and ctypes.sizeof(_lib.EpiFusionParams) == f_size
    assert _lib.EpiFusionBwdParams.feat_dtype.offset == b_off == _lib.EpiFusionBwdParams.grad_vals.offset + 4
    assert _lib.EpiFusionBwdParams.reserved.offset == b_res and ctypes.sizeof(_lib.EpiFusionBwdParams) == b_size
    assert _lib.EPI_ABI_VERSION == ver == 3
    assert (_lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16, _lib.EPI_DTYPE_F16) == (d32, dbf, dh)


def test_bf16_workspace_is_one_fp32_map_smaller(lib):
    """cfg2 pipe shape (N=4, C=256, 64x64, K=64): bf16 maps stage hi planes only, [ref_hi | src_hi] instead of
    [ref_hi | ref_lo | src_hi | src_lo]; fp16 maps are split into (hi, lo) like fp32 ones."""
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = 4, 256, 64, 64, 64
    p.out_stride = (ctypes.c_int64 * 4)(256 * 4096, 4096, 64, 1)
    m = 4 * 256 * 64 * 64 * 4
    sizes = {}
    for name, code in (("f32", _lib.EPI_DTYPE_F32), ("bf16", _lib.EPI_DTYPE_BF16), ("f16", _lib.EPI_DTYPE_F16)):
        p.feat_dtype = code
        assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) > 0                # the pipelined kernel is selected for every dtype
        sizes[name] = lib.epi_fusion_workspace_bytes(ctypes.byref(p))
    assert sizes["f16"] == sizes["f32"]
    assert abs((sizes["f32"] - sizes["bf16"]) - m) < 256, sizes


def test_abi_rejects_unknown_feat_dtype(lib):
    buf = (ctypes.c_float * 4)()
    addr = ctypes.addressof(buf)
    p = _lib.EpiFusionParams()
    p.feat_ref = addr; p.feat_src = addr; p.out = addr; p.P_ref = addr; p.P_src = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 8
    p.downsample = 4.0; p.img_scale = 1.0
    p.feat_dtype = 7
    assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == -1          # EPI_EINVAL
    assert b"feat_dtype" in lib.epi_last_error()
    b = _lib.EpiFusionBwdParams()
    b.feat_ref = addr; b.feat_src = addr; b.attn = addr; b.grad_out = addr; b.P_ref = addr; b.P_src = addr
    b.grad_ref = addr
    b.N, b.C, b.H, b.W, b.K = 1, 8, 8, 8, 8
    b.feat_dtype = 7
    assert lib.epi_fusion_backward_f32(ctypes.byref(b), None) == -1
    assert b"feat_dtype" in lib.epi_last_error()


def _call(a, b, **kw):
    P = torch.zeros(1, 3, 4)
    return epi.epipolar_fusion(a, b, P, P, K=8, **kw)


def test_python_rejects_bad_dtypes():
    x32 = torch.zeros(1, 8, 8, 8)
    with pytest.raises(TypeError, match="same dtype"):
        _call(x32, x32.bfloat16())
    with pytest.raises(TypeError, match="same dtype"):
        _call(x32.half(), x32.bfloat16())
    with pytest.raises(TypeError, match="float32, bfloat16 or float16"):
        _call(x32.double(), x32.double())
    with pytest.raises(TypeError, match="out must be float32"):
        _call(x32.bfloat16(), x32.bfloat16(), out=torch.zeros(1, 8, 8, 8, dtype=torch.float16))
    with pytest.raises(TypeError, match="same dtype"):
        epipolar_fusion_backward(x32, x32.half(), None, None, torch.zeros(1, 8, 8, 8), x32, K=8)
    with pytest.raises(RuntimeError, match="no CPU implementation"):   # a supported dtype on the CPU is still refused
        _call(x32.bfloat16(), x32.bfloat16())
