"""CPU: a bfloat16 / float16 `out` (the output byte of EpiFusionParams.feat_dtype and the out_dtype keyword), checked without a
GPU: the header's encoding, the refusals, the workspace the plan adds for it, the Python refusals and the module's dtype
state.  The library loads without a device; validation and the size queries happen before any CUDA call."""
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
F32, BF16, F16 = _lib.EPI_DTYPE_F32, _lib.EPI_DTYPE_BF16, _lib.EPI_DTYPE_F16
OUT16 = [BF16, F16]


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def al(n):
    return (n + 255) // 256 * 256


def test_encoding_matches_header():
    """EPI_OUT_DTYPE shifts an EPI_DTYPE_* into bits 8-15 of feat_dtype, as a C compile of the header says; the structs keep
    their sizes and offsets (the byte lives in an existing field) and the ABI version stays 3."""
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "enc.c")
        open(c, "w").write(
            '#include <stdio.h>\n#include "%s"\nint main(){printf("%%d %%d %%d %%d %%zu %%zu %%zu %%zu %%zu",'
            ' EPI_OUT_DTYPE(EPI_DTYPE_F32), EPI_OUT_DTYPE(EPI_DTYPE_BF16), EPI_OUT_DTYPE(EPI_DTYPE_F16), EPI_ABI_VERSION,'
            ' sizeof(EpiFusionParams), __builtin_offsetof(EpiFusionParams, feat_dtype), __builtin_offsetof(EpiFusionParams, n_src),'
            ' __builtin_offsetof(EpiFusionParams, cache), sizeof(EpiFusionBwdParams));return 0;}' % HEADER)
        exe = os.path.join(d, "enc")
        subprocess.check_call(["gcc", c, "-o", exe])
        o32, obf, of16, ver, size, off_dt, off_nsrc, off_cache, bsize = map(int, subprocess.check_output([exe]).split())
    assert (o32, obf, of16) == (0, 0x100, 0x200) == tuple(_lib.EPI_OUT_DTYPE(d) for d in (F32, BF16, F16))
    assert ver == _lib.EPI_ABI_VERSION == 3
    P = _lib.EpiFusionParams
    assert (ctypes.sizeof(P), P.feat_dtype.offset, P.n_src.offset, P.cache.offset) == (size, off_dt, off_nsrc, off_cache)
    assert bsize == ctypes.sizeof(_lib.EpiFusionBwdParams) == 328


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def _params(form):
    """params that pass every other check of `form` (pointers to host memory: the call is refused before any is read)"""
    buf = (ctypes.c_float * 4)()
    addr = ctypes.addressof(buf)
    p = _lib.EpiFusionParams()
    p.feat_ref = addr; p.out = addr; p.P_ref = addr
    p.N, p.C, p.H, p.W, p.K = 1, 8, 8, 8, 8
    p.downsample = 4.0; p.img_scale = 1.0
    if form in ("single", "n_src"):
        p.feat_src = addr; p.P_src = addr
        p.n_src = 3 if form == "n_src" else 0
    else:
        p.n_views = 3
    return p, buf


TABLE = np.array([[1], [2], [0]], dtype=np.int32)


def _forward(lib, form, p):
    if form == "table":
        return lib.epi_fusion_view_sources_forward_f32(ctypes.byref(p), TABLE.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 1, None)
    return lib.epi_fusion_forward_f32(ctypes.byref(p), None)


def _sizes(lib, form, p):
    if form == "table":
        t = (TABLE.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 1)
        return lib.epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), *t), lib.epi_fusion_view_sources_cache_bytes(ctypes.byref(p), *t)
    return lib.epi_fusion_workspace_bytes(ctypes.byref(p)), lib.epi_fusion_cache_bytes(ctypes.byref(p))


BAD = {
    "out_byte_3": (F32 | (3 << 8), b"unknown output dtype"),
    "out_byte_255": (BF16 | (255 << 8), b"unknown output dtype"),
    "bit_16": (F32 | (1 << 16), b"bits above 15"),
    "bit_31": (BF16 | _lib.EPI_OUT_DTYPE(BF16) | (1 << 24), b"bits above 15"),
    "negative": (-1, b"bits above 15"),
}


@pytest.mark.parametrize("form", ["single", "n_src", "views", "table"])
@pytest.mark.parametrize("bad", list(BAD))
def test_bad_output_byte_is_einval(lib, form, bad):
    code, msg = BAD[bad]
    p, buf = _params(form)
    p.feat_dtype = code
    assert _forward(lib, form, p) == -1                                  # EPI_EINVAL
    err = lib.epi_last_error()
    assert b"feat_dtype" in err and msg in err, err
    assert _sizes(lib, form, p) == (0, 0)                                # the queries plan nothing for it


@pytest.mark.parametrize("form", ["single", "n_src", "views", "table"])
@pytest.mark.parametrize("od", OUT16, ids=["bf16", "f16"])
def test_valid_output_byte_passes_validation(lib, form, od):
    """a valid output byte gets past validation: the same params without a workspace fail on the workspace, not on the dtype"""
    p, buf = _params(form)
    p.feat_dtype = BF16 | _lib.EPI_OUT_DTYPE(od)
    assert _forward(lib, form, p) == -2                                  # EPI_EWORKSPACE
    assert b"workspace" in lib.epi_last_error()


def test_backward_refuses_an_output_byte(lib):
    """the backward has no `out`: its feat_dtype keeps its one meaning, and an output byte is an unknown feat_dtype"""
    buf = (ctypes.c_float * 4)()
    addr = ctypes.addressof(buf)
    b = _lib.EpiFusionBwdParams()
    b.feat_ref = b.feat_src = b.attn = b.grad_out = b.P_ref = b.P_src = b.grad_ref = addr
    b.N, b.C, b.H, b.W, b.K = 1, 8, 8, 8, 8
    b.feat_dtype = BF16 | _lib.EPI_OUT_DTYPE(BF16)
    assert lib.epi_fusion_backward_f32(ctypes.byref(b), None) == -1
    assert b"feat_dtype" in lib.epi_last_error()


# ---- the workspace ----------------------------------------------------------------------------------------------------------
def _direct(row, cache_bytes):
    """whether the fused kernel stores a float32 `out` itself for this plan-size row: no z, and either a CUDA-core / tile kernel
    (no cache: cache_bytes == 0) or the pipelined kernel with a channels-last, 16-byte-aligned `out` (every C of the sweep is a
    multiple of 4)"""
    variant, dtype, z, cache, n_src, src_cl, out_cl, C, (H, W), K, locs = row
    return not z and (cache_bytes == 0 or out_cl)


def test_plane_added_exactly_where_the_fused_kernel_stored_out(lib):
    """Over a seeded tenth of the plan-size sweep: a 16-bit `out` adds one fp32 plane of the S·N pairs' fused features where
    the float32 plan lets the fused kernel store `out`, and changes no other workspace, cache or backward size."""
    from oracle import make_golden_plan as g
    rows = g.rows()
    pick = np.random.default_rng(0).choice(len(rows), len(rows) // 10, replace=False)
    n_direct = 0
    for i in pick:
        row = rows[i]
        p, b = g._params(row)
        ws32, cb32 = lib.epi_fusion_workspace_bytes(ctypes.byref(p)), lib.epi_fusion_cache_bytes(ctypes.byref(p))
        bw32 = lib.epi_fusion_backward_workspace_bytes(ctypes.byref(b))
        variant, dtype, z, cache, n_src, src_cl, out_cl, C, (H, W), K, locs = row
        plane = al(max(n_src, 1) * g.N * C * H * W * 4)
        direct = _direct(row, cb32)
        n_direct += direct
        for od in OUT16:
            q, _ = g._params(row, feat_dtype=dtype | _lib.EPI_OUT_DTYPE(od))
            ws, cb = lib.epi_fusion_workspace_bytes(ctypes.byref(q)), lib.epi_fusion_cache_bytes(ctypes.byref(q))
            assert cb == cb32, row
            assert ws == ws32 + (plane if direct else 0), (row, od, ws, ws32)
        assert lib.epi_fusion_backward_workspace_bytes(ctypes.byref(b)) == bw32
    assert 0 < n_direct < len(pick)


@pytest.mark.parametrize("z", [False, True], ids=["noz", "z"])
@pytest.mark.parametrize("variant", [_lib.EPI_VARIANT_AUTO, _lib.EPI_VARIANT_WARP], ids=["pipe", "warp"])
@pytest.mark.parametrize("form", ["views", "table"])
def test_views_forms_add_the_pairs_plane(lib, form, variant, z):
    """the views forms: V·S·N pairs' plane (S = V−1, or the table's width) where the fused kernel would have stored `out`"""
    V, N, C, H, W = 3, 2, 64, 32, 32
    S = V - 1 if form == "views" else TABLE.shape[1]
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, 16
    p.ref_stride = (ctypes.c_int64 * 4)(C * H * W, H * W, W, 1)
    p.out_stride = (ctypes.c_int64 * 4)(H * W * C, 1, W * C, C)        # channels-last: the pipe kernel's direct store
    p.feat_ref = p.out = 256
    p.variant, p.n_views = variant, V
    if z:
        p.z_weight_folded = p.z_bias_folded = 256
    ws32, cb32 = _sizes(lib, form, p)
    for od in OUT16:
        p.feat_dtype = _lib.EPI_OUT_DTYPE(od)
        assert _sizes(lib, form, p) == (ws32 + (0 if z else al(V * S * N * C * H * W * 4)), cb32)


# ---- Python -----------------------------------------------------------------------------------------------------------------
def _call(a, b, **kw):
    P = torch.zeros(1, 3, 4)
    return epi.epipolar_fusion(a, b, P, P, K=8, **kw)


def test_python_refusals():
    x = torch.zeros(1, 8, 8, 8)
    xb = x.bfloat16()
    for bad in (torch.float64, torch.int8, "bfloat16", None):
        with pytest.raises(TypeError, match="out_dtype must be"):
            _call(xb, xb, out_dtype=bad)
    with pytest.raises(TypeError, match="out must be bfloat16"):
        _call(xb, xb, out_dtype=torch.bfloat16, out=torch.zeros(1, 8, 8, 8))
    with pytest.raises(TypeError, match="out must be float16"):
        _call(x, x, out_dtype=torch.float16, out=torch.zeros(1, 8, 8, 8, dtype=torch.bfloat16))
    with pytest.raises(TypeError, match="out must be float32"):       # the default keeps its message
        _call(xb, xb, out=torch.zeros(1, 8, 8, 8, dtype=torch.bfloat16))
    f = torch.zeros(3, 1, 8, 8, 8)
    with pytest.raises(TypeError, match="out must be float16"):
        epi.epipolar_fusion_multi(x, f, torch.zeros(1, 3, 4), torch.zeros(3, 1, 3, 4), K=8, out_dtype=torch.float16,
                                  out=torch.zeros(3, 1, 8, 8, 8))
    with pytest.raises(TypeError, match="out_dtype must be"):
        epi.epipolar_fusion_multi(x, f, torch.zeros(1, 3, 4), torch.zeros(3, 1, 3, 4), K=8, out_dtype=torch.float64)
    with pytest.raises(TypeError, match="out must be bfloat16"):
        epi.epipolar_fusion_views(f, torch.zeros(3, 1, 3, 4), K=8, out_dtype=torch.bfloat16, out=torch.zeros(3, 2, 1, 8, 8, 8))
    with pytest.raises(TypeError, match="out_dtype must be"):
        epi.epipolar_fusion_views(f, torch.zeros(3, 1, 3, 4), K=8, out_dtype=torch.float64)
    with pytest.raises(RuntimeError, match="no CPU implementation"):   # valid arguments on the CPU are still refused
        _call(xb, xb, out_dtype=torch.bfloat16, out=torch.zeros(1, 8, 8, 8, dtype=torch.bfloat16))


# ---- the module's dtype -----------------------------------------------------------------------------------------------------
KEYS = sorted(["z.weight", "z.bias", "bn.weight", "bn.bias", "bn.running_mean", "bn.running_var", "bn.num_batches_tracked"])


def test_module_follows_its_cast_dtype():
    m = epi.Epipolar(cfg=epi.cfg_h36m_r50_256())
    assert m.out_dtype == torch.float32 and sorted(m.state_dict().keys()) == KEYS
    assert m.to(torch.bfloat16).out_dtype == torch.bfloat16 and m.z.weight.dtype == torch.bfloat16
    assert m.half().out_dtype == torch.float16
    assert m.bfloat16().out_dtype == torch.bfloat16
    assert m.float().out_dtype == torch.float32
    assert m.to(torch.float16).out_dtype == torch.float16 and sorted(m.state_dict().keys()) == KEYS
    empty = epi.Epipolar(cfg=epi.cfg_h36m_r152_384()).half()              # no parameters: the buffer alone carries the dtype
    assert empty.out_dtype == torch.float16 and list(empty.state_dict().keys()) == []


def test_fp32_checkpoint_loads_into_a_bf16_module():
    src = epi.Epipolar(cfg=epi.cfg_h36m_r50_256())
    torch.manual_seed(0)
    with torch.no_grad():
        for t in (src.z.weight, src.z.bias, src.bn.weight, src.bn.bias, src.bn.running_mean):
            t.copy_(torch.randn_like(t))
        src.bn.running_var.copy_(torch.rand_like(src.bn.running_var) + 0.5)
    sd = src.state_dict()
    m = epi.Epipolar(cfg=epi.cfg_h36m_r50_256()).to(torch.bfloat16)
    m.load_state_dict(sd)                                                  # strict: the same keys, nothing missing
    assert m.out_dtype == torch.bfloat16
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k].to(v.dtype)), k
