"""GPU: bfloat16 / float16 feature maps.  Their values are exact bf16 (hi, lo) pairs of the operand split, so the kernels must
return, bit for bit, what the float32 path returns on the upcast maps — for every kernel variant, layout and epilogue — and the
backward must return float32 gradients rounded once to the maps' dtype."""
import math

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.epipolar import _FusionFn
from oracle import golden_cases as gc
from tests.util import rel_max

pytestmark = pytest.mark.gpu
LOWP = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
VARIANTS = ["auto", "tile", "sector", "warp"]
SCALE = float(epi.make_cfg().EPIPOLAR.SOFTMAXSCALE)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def fold_params(params, bn_eps=1e-5):
    s = params["bn.weight"] / np.sqrt(params["bn.running_var"] + bn_eps)
    wf = (s[:, None] * params["z.weight"].reshape(len(s), -1)).astype(np.float32)
    bf = (s * (params["z.bias"] - params["bn.running_mean"]) + params["bn.bias"]).astype(np.float32)
    return dev(wf), dev(bf)


def case_inputs(name):
    """-> (t1, t2, P1, P2, kwargs of epipolar_fusion) of a golden case, maps as float32 CUDA tensors"""
    cfg, f1, f2, P1, P2, params = gc.build_inputs(name)
    spec = gc.CASES[name]
    kw = dict(K=spec["K"], downsample=cfg.BACKBONE.DOWNSAMPLE, img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
              softmax_scale=cfg.EPIPOLAR.SOFTMAXSCALE, correct_normalize=spec["correct"],
              z_folded=fold_params(params) if params else None, z_residual=spec["zres"])
    return dev(f1), dev(f2), dev(P1), dev(P2), kw


def synthetic_inputs(N, C, H, W, K, seed=0):
    P1, P2 = syn.pairs_from_ring(max(N, 2), int(max(H, W) * 4), seed=seed)
    f1, f2 = syn.features(N, C, H, W, "randn", seed + 1), syn.features(N, C, H, W, "randn", seed + 2)
    return dev(f1), dev(f2), dev(P1[:N].astype(np.float32)), dev(P2[:N].astype(np.float32)), dict(K=K, correct_normalize=True)


def random_z(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, C, generator=g) / math.sqrt(C)).cuda(), (0.1 * torch.randn(C, generator=g)).cuda()


def assert_same_as_fp32(t1, t2, P1, P2, dtype, channels_last=False, **kw):
    """epipolar_fusion on maps of `dtype` vs the float32 call on the same values upcast: all four outputs bit for bit."""
    a, b = t1.to(dtype), t2.to(dtype)
    if channels_last:
        a, b = a.contiguous(memory_format=torch.channels_last), b.contiguous(memory_format=torch.channels_last)
    a32, b32 = a.float(), b.float()                              # .float() keeps the memory format
    kw.setdefault("want_locs", True)
    want = [None if w is None else w.clone(memory_format=torch.preserve_format) for w in epi.epipolar_fusion(a32, b32, P1, P2, **kw)]
    if kw.get("out") is not None:
        kw["out"].fill_(float("nan"))                            # a caller-supplied `out` is shared by both calls
    got = epi.epipolar_fusion(a, b, P1, P2, **kw)
    torch.cuda.synchronize()
    for what, g, w in zip(("out", "corr_pos", "attn", "sample_locs"), got, want):
        if w is None:
            assert g is None
            continue
        assert g.dtype == torch.float32 and g.shape == w.shape, what
        assert torch.equal(g, w), "%s differs: max |diff| %.3g" % (what, (g - w).abs().max().item())
    assert got[0].is_contiguous(memory_format=torch.channels_last) == want[0].is_contiguous(memory_format=torch.channels_last)
    return got


def variant_supported(t1, t2, P1, P2, variant, **kw):
    try:
        epi.epipolar_fusion(t1, t2, P1, P2, variant=variant, **kw)
        return True
    except RuntimeError as e:
        assert "does not support" in str(e)
        return False


# ---- 1. bit-exactness against the float32 path --------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", ["tiny_ring_z", "cfg1_ring", "tiny_randn_krt", "cfg2_r50_256_randn"])
@pytest.mark.parametrize("dtype", LOWP, ids=DT_IDS)
def test_bit_exact_vs_fp32(dtype, name, variant, layout):
    t1, t2, P1, P2, kw = case_inputs(name)
    if not variant_supported(t1, t2, P1, P2, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    assert_same_as_fp32(t1, t2, P1, P2, dtype, channels_last=layout == "channels_last", variant=variant, **kw)


@pytest.mark.parametrize("out_layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("z", ["none", "z", "z+zres"])
@pytest.mark.parametrize("variant", ["auto", "warp"])
@pytest.mark.parametrize("name", ["tiny_ring_z", "cfg2_r50_256_randn"])
@pytest.mark.parametrize("dtype", LOWP, ids=DT_IDS)
def test_residual_and_z_epilogues(dtype, name, variant, z, out_layout):
    """add_ref_residual reads the caller's map in its own dtype in every epilogue: the fused kernel's direct store
    (channels_last out, no z), the transposition pass (NCHW out, no z), the tensor-core z GEMM, and the fp32 z epilogue
    (warp kernel) with and without ZRESIDUAL."""
    t1, t2, P1, P2, kw = case_inputs(name)
    zf = kw.pop("z_folded"); kw.pop("z_residual")
    kw.update(z_folded=None if z == "none" else zf, z_residual=z == "z+zres", add_ref_residual=True, variant=variant)
    if out_layout == "channels_last":
        kw["out"] = torch.empty_like(t1, memory_format=torch.channels_last)
    assert_same_as_fp32(t1, t2, P1, P2, dtype, **kw)


@pytest.mark.parametrize("variant", ["auto", "tile", "warp"])
@pytest.mark.parametrize("dtype", LOWP, ids=DT_IDS)
def test_injected_sample_locs(dtype, variant):
    t1, t2, P1, P2, kw = case_inputs("cfg1_ring")
    locs = epi.epipolar_fusion(t1, t2, P1, P2, want_locs=True, **kw)[3]
    rng = np.random.default_rng(4)
    locs = (locs + dev(rng.uniform(-0.02, 0.02, size=tuple(locs.shape)).astype(np.float32))).contiguous()   # off the fused geometry
    assert_same_as_fp32(t1, t2, P1, P2, dtype, sample_locs_in=locs, variant=variant, **kw)


# (N, C, H, W, K, z): the pipelined kernel's wide channel counts (two query-panel halves), a map above 16384 pixels (row-windowed
# union bitmap), a C % 64 != 0 pipe shape (fp32 z epilogue with the residual), and a C % 8 != 0 shape only the warp kernel takes
SHAPES = {
    "pipe_c320": ((1, 320, 24, 24, 32), "pipe", True),
    "pipe_c512": ((2, 512, 16, 16, 64), "pipe", True),
    "pipe_132x136": ((1, 64, 132, 136, 16), "pipe", False),
    "pipe_c264_fp32z": ((2, 264, 16, 16, 16), "pipe", True),
    "warp_c12": ((2, 12, 12, 20, 16), "warp", False),
}


@pytest.mark.parametrize("add_ref", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", LOWP, ids=DT_IDS)
def test_shape_envelope(dtype, shape, add_ref):
    (N, C, H, W, K), variant, with_z = SHAPES[shape]
    t1, t2, P1, P2, kw = synthetic_inputs(N, C, H, W, K, seed=C)
    if with_z:
        kw.update(z_folded=random_z(C, C), z_residual=True)
    assert_same_as_fp32(t1, t2, P1, P2, dtype, variant=variant, add_ref_residual=add_ref, **kw)
    if variant == "warp":
        assert_same_as_fp32(t1, t2, P1, P2, dtype, variant="auto", add_ref_residual=add_ref, **kw)


# ---- 2. reference semantics under autocast ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg1_ring", "tiny_randn_krt"])
def test_matches_reference_forward_under_autocast(name):
    """The reference layer run under torch.autocast(bfloat16) on bf16 maps computes grid_sample and softmax in float32 on the
    exact bf16 values; the kernel matches it (on the kernel's own sample locations) to the suite's 1e-4."""
    from oracle import torch_port
    cfg, f1, f2, P1, P2, _ = gc.build_inputs(name)
    spec = gc.CASES[name]
    a, b = dev(f1).bfloat16(), dev(f2).bfloat16()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out, corr, attn, locs = epi.epipolar_fusion(a, b, dev(P1), dev(P2), K=spec["K"], softmax_scale=cfg.EPIPOLAR.SOFTMAXSCALE,
                                                    correct_normalize=spec["correct"], want_locs=True)
        r_out, _, r_attn = torch_port.forward(cfg, a, b, P1, P2, locs=locs)
    assert out.dtype == torch.float32 and r_out.dtype == torch.float32
    assert rel_max(out.cpu().numpy(), r_out.cpu().numpy()) < 1e-4
    assert rel_max(attn.cpu().numpy(), r_attn.cpu().numpy()) < 1e-4


# ---- 3. backward --------------------------------------------------------------------------------------------------------
def within_one_ulp(got, ref32, dtype):
    """got (dtype) lies within one ulp of `dtype` of the float32 gradient rounded to dtype"""
    r = ref32.to(dtype).float()
    g = got.float()
    fi = torch.finfo(dtype)
    mag = torch.maximum(r.abs(), g.abs()).clamp_min(fi.tiny)
    ulp = torch.exp2(torch.floor(torch.log2(mag))) * fi.eps
    excess = ((g - r).abs() - ulp).max().item()
    return excess <= 0, excess


BWD_SHAPES = {"vec4_c16": (2, 16, 16, 16, 16), "vec1_c6": (2, 6, 12, 20, 24)}


@pytest.mark.parametrize("other_grad", [("other1", "other2"), ("other1",), ("other2",)], ids=["both", "other1", "other2"])
@pytest.mark.parametrize("shape", list(BWD_SHAPES))
@pytest.mark.parametrize("dtype", LOWP, ids=DT_IDS)
def test_backward_dtype_and_ulp(dtype, shape, other_grad):
    N, C, H, W, K = BWD_SHAPES[shape]
    t1, t2, P1, P2, _ = synthetic_inputs(N, C, H, W, K, seed=7)
    opts = dict(fwd=dict(K=K, downsample=4.0, img_scale=1.0, softmax_scale=SCALE, correct_normalize=True, align_corners=False,
                         want_corr=True, want_locs=False, variant="auto"),
                grad_keys="other1" in other_grad, grad_vals="other2" in other_grad)
    grads = {}
    for dt in (dtype, torch.float32):
        a = t1.to(dtype).to(dt).requires_grad_(True)
        b = t2.to(dtype).to(dt).requires_grad_(True)
        out, _, attn, _ = _FusionFn.apply(a, b, P1, P2, opts)
        assert out.dtype == torch.float32 and attn.dtype == torch.float32
        torch.manual_seed(3)
        w_out, w_attn = torch.randn_like(out), torch.randn_like(attn)
        loss = (out * w_out).sum() + 0.3 * (attn * w_attn).sum()
        grads[dt] = torch.autograd.grad(loss, (a, b))
    for which, g, g32 in zip(("feat_ref", "feat_src"), grads[dtype], grads[torch.float32]):
        assert g.dtype == dtype, which
        ok, excess = within_one_ulp(g, g32, dtype)
        assert ok, "%s: %.3g beyond one ulp" % (which, excess)
        assert g32.abs().max().item() > 0, which


# ---- 4. persistent cache ------------------------------------------------------------------------------------------------
def test_fusion_state_across_dtypes():
    """one FusionState driven fp32 -> bf16 -> bf16 -> fp32: the plan (operand planes, kernel form) follows the dtype"""
    t1, t2, P1, P2, kw = case_inputs("cfg2_r50_256_randn")
    maps = {torch.float32: (t1, t2), torch.bfloat16: (t1.bfloat16(), t2.bfloat16())}
    want = {dt: epi.epipolar_fusion(*m, P1, P2, **kw) for dt, m in maps.items()}
    state = epi.FusionState()
    for dt in (torch.float32, torch.bfloat16, torch.bfloat16, torch.float32):
        got = epi.epipolar_fusion(*maps[dt], P1, P2, state=state, **kw)
        for g, w in zip(got, want[dt]):
            assert (g is None and w is None) or torch.equal(g, w), dt


# ---- 5. the module under autocast ---------------------------------------------------------------------------------------
def _module_inputs(cfg, N=2, seed=11):
    C, (H, W) = cfg.KEYPOINT.NFEATS, cfg.KEYPOINT.HEATMAP_SIZE
    img = int(max(H, W) * cfg.BACKBONE.DOWNSAMPLE)
    P1, P2 = syn.pairs_from_ring(max(N, 2), img, seed=seed)
    f1, f2 = syn.features(N, C, H, W, "relu_smooth", seed), syn.features(N, C, H, W, "relu_smooth", seed + 1)
    return dev(f1), dev(f2), dev(P1[:N].astype(np.float32)), dev(P2[:N].astype(np.float32))


def test_module_eval_under_autocast_matches_fp32():
    cfg = epi.cfg_h36m_r50_256()
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    params = syn.z_bn_params(cfg.KEYPOINT.NFEATS, 5)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    t1, t2, P1, P2 = _module_inputs(cfg)
    a, b = t1.bfloat16(), t2.bfloat16()
    with torch.no_grad():
        want = m(a.float(), b.float(), P1, P2)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got = m(a, b, P1, P2)
            got2 = m(a, b, P1, P2)                       # the module's persistent state, second call
    for g, g2, w in zip(got, got2, want):
        if w is None:
            continue
        assert g.dtype == torch.float32
        assert torch.equal(g, w) and torch.equal(g2, w)


def test_module_trains_under_autocast():
    cfg = epi.cfg_h36m_r50_256()
    m = epi.Epipolar(cfg=cfg).cuda().train()
    params = syn.z_bn_params(cfg.KEYPOINT.NFEATS, 6)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    t1, t2, P1, P2 = _module_inputs(cfg, seed=12)
    a = t1.bfloat16().requires_grad_(True)
    b = t2.bfloat16().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out, corr, attn, _ = m(a, b, P1, P2)
        loss = out.float().square().mean() + attn.float().mean()
    loss.backward()
    for name, g in (("feat1", a.grad), ("feat2", b.grad), ("z.weight", m.z.weight.grad), ("bn.weight", m.bn.weight.grad)):
        assert g is not None and torch.isfinite(g).all(), name
    assert a.grad.dtype == torch.bfloat16 and b.grad.dtype == torch.bfloat16
    assert a.grad.abs().max().item() > 0 and b.grad.abs().max().item() > 0
