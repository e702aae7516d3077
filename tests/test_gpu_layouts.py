"""GPU: the kernels on odd-sized maps and on the strided, offset and broadcast views the ABI accepts, against float64.

  1. Odd maps (H·W % 4 != 0): every vector path the kernels take on even maps has a scalar tail here (the staging tiles,
     the z GEMM's last pixel tile and non-vector epilogue, the transposition pass).  Each case asserts the plan it is meant to
     reach (kernel launches; the pipelined kernel is the only one with a cache), then out / attn / corr_pos against the fp64
     restatement on the kernel's own locations, and the locations against the fp64 reference geometry.
  2. Views: maps and `out` as batch steps, channel slices, crops, odd element offsets, transposes, channel-slices of
     channels-last buffers (16-byte aligned or not) and a broadcast reference, padded with NaN.  Every result must be bit for
     bit what the same call on `.contiguous()` copies gives, and nothing around a view may be written.
  3. Backward on views, default and deterministic, against the fp64 autograd restatement of tests/test_gpu_backward.py.

The calls go through the test-local driver (tests/util.py), so the test owns every buffer."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, synthetic as syn
from oracle import epipolar_oracle as eo
from tests.util import bwd_params, check_corr, fp64_reference, fusion_params, launch, px_err, rel_max, workspace_bytes

pytestmark = pytest.mark.gpu
TOL = 1e-4
SCALE = 0.125
LOWP = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


def cameras(N, H, W, S=1, seed=0):
    """ring cameras: P1 [N,3,4], P2 [S·N,3,4] (pair s·N + n: reference n against another view of the ring)"""
    KRT = syn.ring_cameras(N + S, 4 * max(H, W), seed=seed, jitter=20.0)
    P2 = np.concatenate([KRT[[(n + 1 + s) % (N + S) for n in range(N)]] for s in range(S)])
    return KRT[:N].astype(np.float32), P2.astype(np.float32)


def z_weights(C, seed=3):
    """(raw z / BN parameters, (Wf, bf) folded on the host in fp64 and rounded to fp32 on the device)"""
    prm = syn.z_bn_params(C, seed)
    s = prm["bn.weight"].astype(np.float64) / np.sqrt(prm["bn.running_var"].astype(np.float64) + 1e-5)
    wf = s[:, None] * prm["z.weight"].reshape(C, C).astype(np.float64)
    bf = s * (prm["z.bias"].astype(np.float64) - prm["bn.running_mean"]) + prm["bn.bias"]
    return prm, (torch.from_numpy(wf.astype(np.float32)).cuda(), torch.from_numpy(bf.astype(np.float32)).cuda())


@functools.lru_cache(maxsize=None)
def inputs(N, C, H, W, S=1, dtype="f32", seed=0):
    """f1 [N,C,H,W], f2 [S·N,C,H,W] on the device in `dtype` (contiguous NCHW), P1, P2 as numpy"""
    f1 = torch.from_numpy(syn.features(N, C, H, W, "randn", seed + 1)).cuda().to(LOWP[dtype])
    f2 = torch.from_numpy(syn.features(S * N, C, H, W, "randn", seed + 2)).cuda().to(LOWP[dtype])
    return f1, f2, *cameras(N, H, W, S, seed)


def forward(f1, f2, P1, P2, K, out=None, **kw):
    """one forward through the driver with fresh attn / corr_pos / sample_locs -> dict of results, launches, plan facts"""
    NP, C, H, W = f2.shape
    if out is None:
        out = torch.empty((NP, C, H, W), device="cuda")
    attn = torch.empty((NP, K, H, W), device="cuda")
    corr = torch.empty((NP, H, W, 2), device="cuda")
    locs = torch.empty((K, NP, H, W, 2), device="cuda")
    P1, P2 = torch.from_numpy(P1).cuda(), torch.from_numpy(P2).cuda()      # held until the call has finished
    p = fusion_params(f1, f2, out, K=K, P1=P1, P2=P2, attn=attn, corr=corr, locs_out=locs, **kw)
    nbytes = workspace_bytes(p)
    ws = torch.empty(nbytes, device="cuda", dtype=torch.uint8) if nbytes else None
    pipe = _lib.load().epi_fusion_cache_bytes(ctypes.byref(p)) > 0
    n = launch(p, ws)
    return dict(out=out, attn=attn, corr=corr, locs=locs, launches=n, pipe=pipe, ws=nbytes)


def reference(f1, f2, locs, S, correct, align_corners, pixels, z=None, z_residual=False, add_ref=False):
    """fp64 out [NP,C,P] (with the z / BN epilogue of oracle.epipolar_oracle and the residual), attn [NP,K,P], corr [NP,P,2]"""
    f1 = np.concatenate([f1.float().cpu().numpy()] * S)
    f2 = f2.float().cpu().numpy()
    ro, ra, rc = fp64_reference(f1, f2, locs, SCALE, correct, align_corners, pixels)
    if z is not None:
        ro = eo.z_epilogue(ro[..., None], z, z_residual)[..., 0]
    if add_ref:
        NP, C = f1.shape[:2]
        ro = ro + f1.reshape(NP, C, -1)[np.arange(NP)[:, None], :, pixels].transpose(0, 2, 1)
    return ro, ra, rc


def subsample(NP, HW, n_px=256, seed=0):
    if HW <= 1100:
        return np.broadcast_to(np.arange(HW), (NP, HW))
    rng = np.random.default_rng(seed)
    return np.stack([np.sort(rng.choice(HW, n_px, replace=False)) for _ in range(NP)])


def check_against_fp64(r, f1, f2, P1, P2, K, S, correct=True, align_corners=False, z=None, z_residual=False, add_ref=False):
    NP, C, H, W = f2.shape
    locs = r["locs"].cpu().numpy()
    pixels = subsample(NP, H * W)
    ro, ra, rc = reference(f1, f2, locs, S, correct, align_corners, pixels, z, z_residual, add_ref)
    idx = np.arange(NP)[:, None]
    out = r["out"].cpu().numpy().reshape(NP, C, H * W)[idx, :, pixels].transpose(0, 2, 1)
    attn = r["attn"].cpu().numpy().reshape(NP, K, H * W)[idx, :, pixels].transpose(0, 2, 1)
    corr = r["corr"].cpu().numpy().reshape(NP, H * W, 2)[idx, pixels]
    assert rel_max(out, ro) < TOL, rel_max(out, ro)
    assert rel_max(attn, ra) < TOL, rel_max(attn, ra)
    for n in range(NP):
        ys, xs = np.divmod(pixels[n], W)
        check_corr(corr[n], rc[n], ra[n], locs[:, n, ys, xs], H, W, correct)
    # the geometry on the odd map: the same far set as the fp64 reference geometry, and every emitted location within 1e-3
    # feature px of it, or as close as the reference's own fp32 geometry gets (161x163: 6e-3 px where a line meets the border
    # at a grazing angle)
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=correct))
    ref64 = eo.sample_locs(cfg, np.concatenate([P1] * S), P2, H, W, K, np.float64)
    err, far_ok = px_err(locs, ref64, H, W)
    ref_err, _ = px_err(eo.sample_locs(cfg, np.concatenate([P1] * S), P2, H, W, K, np.float32), ref64, H, W)
    assert far_ok and err < max(1e-3, ref_err), (err, far_ok, ref_err)


# ---------------------------------------------------------------------------------------------------------------------
# 1. odd maps
SHAPES = {
    "13x21": (2, 64, 13, 21, 16),       # HW = 273: a partial 64-pixel item, a 17-pixel last z tile
    "31x33": (2, 256, 31, 33, 64),      # production C / K, HW = 1023: a 127-pixel last z tile, non-vector z epilogue
    "17x19": (1, 512, 17, 19, 64),      # two query halves, 32-pixel items, four 128-channel z output blocks
    "15x17": (2, 264, 15, 17, 16),      # C % 64 != 0: the fp32 z epilogue behind the pipelined kernel
    "127x129": (1, 64, 127, 129, 64),   # K = 64 on a 129-pixel side: automatic selection takes sector tiles, 16383 pixels
    "161x163": (1, 32, 161, 163, 16),   # above 16384 pixels: row-windowed union, pixel order in a launch of its own
    "11x13": (2, 12, 11, 13, 16),       # C % 8 != 0: CUDA-core kernel
    "7x9": (1, 516, 7, 9, 32),          # C > 512: CUDA-core kernel
}
# (map, variant, dtype, maps' layout, out layout, epilogue, n_src, align_corners, plan, launches)
# plan: pipe_direct (the fused kernel writes out), pipe_unstage (+ transposition pass), pipe_zgemm (+ tensor-core z GEMM),
# pipe_zfp32 (+ fp32 z epilogue), +refcopy_after (a fp32 copy of the low-precision reference for that epilogue's residual),
# +order_apart (the pixel order in a launch of its own); sector, tile, warp (+ their staging, reference copy and z launches)
ODD = [
    ("13x21", "auto", "f32", "nchw", "nchw", "none", 1, False, "pipe_unstage", 3),
    ("13x21", "auto", "bf16", "cl", "cl", "add_ref", 1, False, "pipe_direct", 2),
    ("13x21", "auto", "f16", "nchw", "cl", "z", 1, False, "pipe_zgemm", 3),
    ("13x21", "auto", "f32", "cl", "nchw", "zres_add_ref", 1, False, "pipe_zgemm", 3),
    ("13x21", "auto", "f32", "nchw", "nchw", "zres", 3, False, "pipe_zgemm", 3),
    ("13x21", "auto", "f32", "nchw", "cl", "none", 1, True, "pipe_direct", 2),
    ("13x21", "sector", "f32", "nchw", "nchw", "none", 1, False, "sector", 4),
    ("13x21", "tile", "bf16", "cl", "cl", "add_ref", 1, False, "tile", 3),
    ("13x21", "warp", "f16", "nchw", "nchw", "z", 1, False, "warp", 4),
    ("13x21", "warp", "f32", "cl", "cl", "none", 1, False, "warp", 1),
    ("31x33", "auto", "f32", "nchw", "nchw", "z", 1, False, "pipe_zgemm", 3),
    ("31x33", "auto", "bf16", "cl", "nchw", "add_ref", 1, False, "pipe_unstage", 3),
    ("31x33", "auto", "f16", "nchw", "cl", "none", 1, False, "pipe_direct", 2),
    ("17x19", "auto", "f32", "nchw", "nchw", "zres", 1, False, "pipe_zgemm", 3),
    ("17x19", "auto", "bf16", "cl", "cl", "none", 1, False, "pipe_direct", 2),
    ("15x17", "auto", "f32", "nchw", "nchw", "z", 1, False, "pipe_zfp32", 3),
    ("15x17", "auto", "bf16", "nchw", "nchw", "zres_add_ref", 1, False, "pipe_zfp32+refcopy_after", 4),
    ("15x17", "auto", "f16", "cl", "cl", "add_ref", 1, False, "pipe_direct", 2),
    ("127x129", "auto", "f32", "nchw", "nchw", "none", 1, False, "sector", 4),
    ("127x129", "auto", "bf16", "cl", "cl", "z", 1, False, "sector", 6),
    ("161x163", "auto", "f32", "nchw", "nchw", "none", 1, False, "pipe_unstage+order_apart", 4),
    ("161x163", "auto", "bf16", "cl", "cl", "add_ref", 1, False, "pipe_direct+order_apart", 3),
    ("11x13", "auto", "f32", "nchw", "nchw", "add_ref", 1, False, "warp", 2),
    ("11x13", "auto", "bf16", "cl", "cl", "none", 1, False, "warp", 3),
    ("7x9", "auto", "f32", "cl", "nchw", "z", 1, False, "warp", 2),
    ("7x9", "auto", "f16", "nchw", "cl", "zres_add_ref", 1, False, "warp", 4),
]
ODD_PARAMS = [pytest.param(*c, id="%s-%s-%s-%s-%s-%s%s%s-%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "-nsrc3" if c[6] > 1 else "",
                                                                "-align" if c[7] else "", c[8])) for c in ODD]


def to_layout(t, layout):
    return t.contiguous(memory_format=torch.channels_last) if layout == "cl" else t.contiguous()


@pytest.mark.parametrize("shape,variant,dtype,in_layout,out_layout,epilogue,S,align,plan,launches", ODD_PARAMS)
def test_odd_maps_vs_fp64(shape, variant, dtype, in_layout, out_layout, epilogue, S, align, plan, launches):
    N, C, H, W, K = SHAPES[shape]
    f1, f2, P1, P2 = inputs(N, C, H, W, S, dtype)
    f1, f2 = to_layout(f1, in_layout), to_layout(f2, in_layout)
    out = to_layout(torch.empty((S * N, C, H, W), device="cuda"), out_layout)
    prm, z = z_weights(C) if "z" in epilogue else (None, None)
    kw = dict(z=z, z_residual="zres" in epilogue, add_ref="add_ref" in epilogue, variant=variant, n_src=S if S > 1 else 0,
              align_corners=align)
    r = forward(f1, f2, P1, P2, K, out=out, **kw)
    assert (r["launches"], r["pipe"]) == (launches, plan.startswith("pipe")), (r["launches"], r["pipe"])
    check_against_fp64(r, f1, f2, P1, P2, K, S, align_corners=align, z=prm, z_residual=kw["z_residual"], add_ref=kw["add_ref"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. views
def padded(shape, dtype):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def map_view(kind, x):
    """a view of a NaN-padded buffer holding x's values (x: contiguous [N,C,H,W]) -> (view, buffer)"""
    N, C, H, W = x.shape
    if kind == "batch_step":
        buf = padded((2 * N, C, H, W), x.dtype); v = buf[::2]
    elif kind == "channel_slice":             # base offset 3·H·W elements: only element-aligned when H·W is odd
        buf = padded((N, C + 6, H, W), x.dtype); v = buf[:, 3:3 + C]
    elif kind == "crop":
        buf = padded((N, C, H + 3, W + 5), x.dtype); v = buf[..., 1:1 + H, 2:2 + W]
    elif kind == "offset":
        buf = padded((x.numel() + 1,), x.dtype); v = buf[1:1 + x.numel()].view(N, C, H, W)
    elif kind == "transposed":
        buf = padded((N, C, W, H), x.dtype); v = buf.transpose(2, 3)
    elif kind == "cl_slice_aligned":          # channels of a channels-last buffer, 8 elements in: 16-byte aligned for every dtype
        buf = padded((N, H, W, C + 8), x.dtype); v = buf[..., 8:8 + C].permute(0, 3, 1, 2)
    elif kind == "cl_slice_misaligned":
        buf = padded((N, H, W, C + 8), x.dtype); v = buf[..., 1:1 + C].permute(0, 3, 1, 2)
    else:
        raise ValueError(kind)
    v.copy_(x)
    return v, buf


MAP_VIEWS = ["batch_step", "channel_slice", "crop", "offset", "transposed", "cl_slice_aligned", "cl_slice_misaligned",
             "expand_ref"]
OUT_VIEWS = ["out_cl_aligned", "out_cl_misaligned", "out_crop", "out_batch_step"]


def untouched_outside(buf, before, view, view_before):
    """every element of `buf` outside `view` still holds its bits from before the call"""
    got = view.clone()
    view.copy_(view_before)
    same = torch.equal(buf.view(torch.int32) if buf.dtype == torch.float32 else buf.view(torch.int16),
                       before.view(torch.int32) if buf.dtype == torch.float32 else before.view(torch.int16))
    view.copy_(got)
    return same


@functools.lru_cache(maxsize=None)
def contiguous_result(shape, dtype, add_ref):
    N, C, H, W, K = SHAPES[shape]
    f1, f2, P1, P2 = inputs(N, C, H, W, 1, dtype)
    r = forward(f1, f2, P1, P2, K, add_ref=add_ref)
    check_against_fp64(r, f1, f2, P1, P2, K, 1, add_ref=add_ref)
    return r


def assert_same_bits(got, want, what=("out", "attn", "corr", "locs")):
    for k in what:
        g, w = got[k].contiguous(), want[k].contiguous()
        assert torch.equal(g.view(torch.int32), w.view(torch.int32)), k


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("kind", MAP_VIEWS)
@pytest.mark.parametrize("shape", ["13x21", "31x33"])
def test_map_views_equal_contiguous(shape, kind, dtype):
    """Both maps as the same kind of view (the reference only, broadcast over the batch, for expand_ref): the pipelined
    kernel stages every layout into the same bf16 (hi, lo) planes, so all four outputs are bit for bit the contiguous
    call's, and the padding of the views is never read (it is NaN, which would reach the results)."""
    N, C, H, W, K = SHAPES[shape]
    f1, f2, P1, P2 = inputs(N, C, H, W, 1, dtype)
    add_ref = kind in ("crop", "transposed", "expand_ref")           # the residual read through the view's strides too
    if kind == "expand_ref":
        v1, v2 = f1[:1].expand(N, C, H, W), f2
        assert v1.stride(0) == 0
        want = forward(v1.contiguous(), f2, P1, P2, K, add_ref=add_ref)
        check_against_fp64(want, v1.contiguous(), f2, P1, P2, K, 1, add_ref=add_ref)
    else:
        (v1, b1), (v2, b2) = map_view(kind, f1), map_view(kind, f2)
        want = contiguous_result(shape, dtype, add_ref)
    if kind == "channel_slice" and dtype == "f32":
        assert (v1.data_ptr() % 16 != 0) == (H * W % 2 == 1)
    got = forward(v1, v2, P1, P2, K, add_ref=add_ref)
    assert got["pipe"] and got["launches"] == want["launches"]
    assert_same_bits(got, want)


def out_view(kind, NP, C, H, W):
    if kind == "out_cl_aligned":
        buf = padded((NP, H, W, C + 8), torch.float32); v = buf[..., 8:8 + C].permute(0, 3, 1, 2)
    elif kind == "out_cl_misaligned":           # strides are multiples of 4, the base is 4 bytes off a 16-byte boundary
        buf = padded((NP, H, W, C + 4), torch.float32); v = buf[..., 1:1 + C].permute(0, 3, 1, 2)
    elif kind == "out_crop":
        buf = padded((NP, C, H + 2, W + 2), torch.float32); v = buf[:, :, 1:1 + H, 1:1 + W]
    else:
        buf = padded((2 * NP, C, H, W), torch.float32); v = buf[::2]
    return v, buf


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("kind", OUT_VIEWS)
@pytest.mark.parametrize("shape", ["13x21", "31x33"])
def test_out_views_equal_contiguous(shape, kind, dtype):
    """`out` as a view (with the reference residual, so that the fused kernel's direct store adds it itself): the values are
    the same fp32 sums whoever stores them, so `out` is bit for bit the contiguous call's, and no element of the buffer
    around the view is written.  The misaligned channels-last `out` runs only after the pure workspace query has shown
    that it takes the transposition pass."""
    N, C, H, W, K = SHAPES[shape]
    f1, f2, P1, P2 = inputs(N, C, H, W, 1, dtype)
    v, buf = out_view(kind, N, C, H, W)
    if kind == "out_cl_misaligned":
        assert v.data_ptr() % 16 == 4 and all(s % 4 == 0 for s in (v.stride(0), v.stride(2), v.stride(3))) and v.stride(1) == 1
        aligned = buf[..., 4:4 + C].permute(0, 3, 1, 2)           # the same strides at a 16-byte-aligned base
        p_mis = fusion_params(f1, f2, v, K=K, add_ref=True)
        p_al = fusion_params(f1, f2, aligned, K=K, add_ref=True)
        assert workspace_bytes(p_mis) == workspace_bytes(p_al) + -(-N * C * H * W * 4 // 256) * 256, \
            "a misaligned out must take the transposition pass"
    before = buf.clone()
    got = forward(f1, f2, P1, P2, K, out=v, add_ref=True)
    want = contiguous_result(shape, dtype, True)
    assert got["pipe"]
    assert got["launches"] == (2 if kind == "out_cl_aligned" else 3)
    assert_same_bits(dict(got, out=v), want)
    assert untouched_outside(buf, before, v, before.as_strided(v.shape, v.stride(), v.storage_offset()))


# ---------------------------------------------------------------------------------------------------------------------
# 3. backward on views
BWD = [  # (N, C, H, W, K), dtype, deterministic, view of feat_ref / feat_src / grad_out
    ((2, 17, 11, 13, 40), "f32", False, "none"),
    ((2, 17, 11, 13, 40), "bf16", True, "channel_slice"),
    ((2, 17, 11, 13, 40), "f16", False, "crop"),
    ((2, 17, 11, 13, 40), "f32", True, "transposed"),
    ((2, 64, 13, 21, 48), "f32", True, "offset"),
    ((2, 64, 13, 21, 48), "bf16", False, "cl_slice_misaligned"),
    ((2, 64, 13, 21, 48), "f16", True, "batch_step"),
    ((2, 64, 13, 21, 48), "f32", False, "cl_slice_aligned"),
    ((1, 256, 31, 33, 64), "f32", True, "crop"),
    ((1, 256, 31, 33, 64), "bf16", True, "none"),
    ((1, 256, 31, 33, 64), "f16", False, "channel_slice"),
    ((1, 256, 31, 33, 64), "f32", False, "batch_step"),
]
BWD_PARAMS = [pytest.param(*c, id="%s-%s-%s-%s" % ("x".join(map(str, c[0])), c[1], "det" if c[2] else "default", c[3]))
              for c in BWD]


def backward(f1, f2, attn, g_out, K, locs, deterministic):
    g_ref, g_src = torch.empty(f1.shape, device="cuda", dtype=f1.dtype), torch.empty(f2.shape, device="cuda", dtype=f2.dtype)
    b = bwd_params(f1, f2, attn, g_out, K=K, locs_in=locs, grad_ref=g_ref, grad_src=g_src, deterministic=deterministic)
    nbytes = _lib.load().epi_fusion_backward_workspace_bytes(ctypes.byref(b))
    launch(b, torch.empty(nbytes, device="cuda", dtype=torch.uint8), backward=True)
    return g_ref, g_src


@pytest.mark.parametrize("shape,dtype,det,kind", BWD_PARAMS)
def test_backward_views_vs_fp64(shape, dtype, det, kind):
    from tests.test_gpu_backward import reference_grads
    N, C, H, W, K = shape
    f1, f2, P1, P2 = inputs(N, C, H, W, 1, dtype, seed=4)
    fwd = forward(f1, f2, P1, P2, K)
    torch.manual_seed(5)
    g_out = torch.randn((N, C, H, W), device="cuda")
    if kind == "none":
        v1, v2, vg = f1, f2, g_out
    else:
        v1, v2, vg = map_view(kind, f1)[0], map_view(kind, f2)[0], map_view(kind, g_out)[0]
    g1, g2 = backward(v1, v2, fwd["attn"], vg, K, fwd["locs"], det)
    c1, c2 = backward(f1, f2, fwd["attn"], g_out, K, fwd["locs"], det)
    if det:                        # bit-reproducible: whatever the layouts, and from run to run
        r1, r2 = backward(v1, v2, fwd["attn"], vg, K, fwd["locs"], det)
        for a, b in ((g1, c1), (g2, c2), (g1, r1), (g2, r2)):
            assert torch.equal(a.view(torch.int16 if a.dtype != torch.float32 else torch.int32),
                               b.view(torch.int16 if b.dtype != torch.float32 else torch.int32))
    else:                          # dL/dfeat_ref is order-fixed on both paths
        assert torch.equal(g1, c1)
    _, e1, e2 = reference_grads(f1.float(), f2.float(), fwd["locs"], g_out, None)
    tol = TOL + (torch.finfo(LOWP[dtype]).eps if dtype != "f32" else 0.0)        # + the rounding to the maps' dtype
    assert rel_max(g1.float().cpu().numpy(), e1.cpu().numpy()) < tol
    assert rel_max(g2.float().cpu().numpy(), e2.cpu().numpy()) < tol
