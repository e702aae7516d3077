"""GPU: a bfloat16 / float16 `out` (out_dtype=, the output byte of EpiFusionParams.feat_dtype).  Every call must return, as its
`out`, the same call's float32 `out` rounded once (`.to(dtype)`, round to nearest even), bit for bit, and attn, corr_pos and
sample_locs bit for bit as the float32 call returns them — over the forms, epilogues, kernel variants, map dtypes and `out`
layouts.  The driver-level cases put `out` between guard bands and run over a poisoned workspace, as tests/test_gpu_buffers.py
does.  The module cases cast an Epipolar layer to bfloat16 / float16 and compare it with the float32 layer on the upcast
parameters, in eval and in a training step."""

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from epipolar_transformers_b200 import epipolar as epimod
from tests.test_gpu_buffers import Guarded, int_bits, poisoned
from tests.test_gpu_views import random_z, view_inputs
from tests.util import fusion_params, launch, workspace_bytes

pytestmark = pytest.mark.gpu
OUT16 = [torch.bfloat16, torch.float16]
OD_IDS = ["out_bf16", "out_f16"]
MAPS = [torch.float32, torch.bfloat16, torch.float16]
NAMES = ("out", "corr_pos", "attn", "sample_locs")
V = 4
TABLE = [[(v + 1) % V] for v in range(V)]          # each view with its neighbour on the ring (S = 1)


bits = int_bits


def assert_rounded(got, want, od):
    """got: the call with out_dtype=od; want: the same call in float32"""
    g, w = got[0], want[0]
    assert g.dtype == od and w.dtype == torch.float32 and g.shape == w.shape
    assert g.is_contiguous(memory_format=torch.channels_last) == w.is_contiguous(memory_format=torch.channels_last)
    r = w.to(od)
    if not torch.equal(bits(g), bits(r)):
        bad = (bits(g) != bits(r)).sum().item()
        pytest.fail("out: %d of %d elements differ from the float32 out rounded to %s (max |diff| %.3g)" % (
            bad, g.numel(), od, (g.float() - r.float()).abs().max().item()))
    for name, a, b in zip(NAMES[1:], got[1:], want[1:]):
        assert (a is None) == (b is None), name
        if a is not None:
            assert a.dtype == torch.float32 and torch.equal(bits(a), bits(b)), "%s differs from the float32 call" % name


def call(form, feats, P, **kw):
    """one call of `form` on views feats [V,N,C,H,W] / P [V,N,3,4]"""
    kw.setdefault("want_locs", True)
    if form == "single":
        return epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], **kw)
    if form == "n_src3":
        return epi.epipolar_fusion_multi(feats[0], feats[1:4], P[0], P[1:4], **kw)
    if form == "views":
        return epi.epipolar_fusion_views(feats, P, **kw)
    if form == "table":
        return epi.epipolar_fusion_views(feats, P, sources=TABLE, **kw)
    raise ValueError(form)


def compare(form, feats, P, od, **kw):
    want = [None if t is None else t.clone() for t in call(form, feats, P, **kw)]
    got = call(form, feats, P, out_dtype=od, **kw)
    torch.cuda.synchronize()
    assert_rounded(got, want, od)
    return got


def epilogue_kw(epilogue, C):
    z = random_z(C, 5) if epilogue.startswith("z") else None
    return dict(z_folded=z, z_residual=epilogue == "z+zres", add_ref_residual=epilogue in ("add_ref", "z+res"))


EPILOGUES = ["none", "add_ref", "z", "z+zres", "z+res"]


# ---- 1. every form x epilogue, at the z GEMM's C and the fp32 z epilogue's C ------------------------------------------------
@pytest.mark.parametrize("od", OUT16, ids=OD_IDS)
@pytest.mark.parametrize("C", [256, 264], ids=["c256_zgemm", "c264_zfp32"])
@pytest.mark.parametrize("epilogue", EPILOGUES)
@pytest.mark.parametrize("form", ["single", "n_src3", "views", "table"])
def test_forms_and_epilogues(form, epilogue, C, od):
    i = ["single", "n_src3", "views", "table"].index(form) + EPILOGUES.index(epilogue)
    mdt = MAPS[i % 3]                                             # every map dtype meets every form and epilogue
    feats, P, kw = view_inputs(V, 2, C, 15, 17, 16, seed=i)
    compare(form, feats.to(mdt), P, od, **kw, **epilogue_kw(epilogue, C))


# ---- 2. kernel variants x map dtypes, with and without the caller's residual and the z epilogue -----------------------------
@pytest.mark.parametrize("od", OUT16, ids=OD_IDS)
@pytest.mark.parametrize("epilogue", ["none", "add_ref", "z+zres"])
@pytest.mark.parametrize("mdt", MAPS, ids=["maps_f32", "maps_bf16", "maps_f16"])
@pytest.mark.parametrize("variant", ["auto", "pipe", "tile", "sector", "warp"])
def test_variants(variant, mdt, epilogue, od):
    feats, P, kw = view_inputs(2, 2, 64, 13, 21, 16, seed=7)
    compare("single", feats.to(mdt), P, od, variant=variant, **kw, **epilogue_kw(epilogue, 64))


@pytest.mark.parametrize("variant", ["pipe", "sector", "warp"])
@pytest.mark.parametrize("form", ["views", "table"])
def test_views_forms_on_each_kernel(form, variant):
    feats, P, kw = view_inputs(V, 1, 64, 13, 21, 16, seed=9)
    compare(form, feats.to(torch.bfloat16), P, torch.bfloat16, variant=variant, add_ref_residual=True, **kw)


# ---- 3. `out` layouts -------------------------------------------------------------------------------------------------------
def out_buffer(layout, shape, od):
    """-> (out view, the whole buffer) of dtype od, the buffer filled with NaN around the view"""
    NP, C, H, W = shape
    if layout == "nchw":
        buf = torch.full(shape, float("nan"), device="cuda", dtype=od); return buf, buf
    if layout == "channels_last":
        buf = torch.full((NP, H, W, C), float("nan"), device="cuda", dtype=od); return buf.permute(0, 3, 1, 2), buf
    if layout == "strided":                     # every other item, a crop of a wider row, channels at twice the pitch
        buf = torch.full((2 * NP, 2 * C, H, W + 3), float("nan"), device="cuda", dtype=od)
        return buf[::2, ::2, :, 1:W + 1], buf
    if layout == "misaligned2":                 # contiguous NCHW whose base is one 2-byte element off a 4-byte boundary
        buf = torch.full((NP * C * H * W + 1,), float("nan"), device="cuda", dtype=od)
        v = buf[1:].view(shape)
        assert v.data_ptr() % 4 == 2
        return v, buf
    raise ValueError(layout)


@pytest.mark.parametrize("od", OUT16, ids=OD_IDS)
@pytest.mark.parametrize("epilogue", ["none", "add_ref", "z+res"])
@pytest.mark.parametrize("C", [256, 264], ids=["c256", "c264"])
@pytest.mark.parametrize("layout", ["nchw", "channels_last", "strided", "misaligned2"])
def test_out_layouts(layout, C, epilogue, od):
    feats, P, kw = view_inputs(2, 2, C, 16, 20, 16, seed=11)
    f1, f2 = feats[0].to(torch.bfloat16), feats[1].to(torch.bfloat16)
    kw.update(want_locs=True, **epilogue_kw(epilogue, C))
    want = epi.epipolar_fusion(f1, f2, P[0], P[1], **kw)
    out, buf = out_buffer(layout, tuple(f1.shape), od)
    before = bits(buf).clone()
    got = epi.epipolar_fusion(f1, f2, P[0], P[1], out=out, out_dtype=od, **kw)
    torch.cuda.synchronize()
    assert got[0] is out
    assert torch.equal(bits(out), bits(want[0].to(od))), "out differs from the float32 out rounded"
    for a, b in zip(got[1:], want[1:]):
        assert torch.equal(bits(a), bits(b))
    out.copy_(torch.full_like(out, float("nan")))                 # the view back to its old contents: the buffer must be too
    assert torch.equal(bits(buf), before), "an element outside the `out` view was written"


# ---- 4. guard bands and a poisoned workspace (driver level) -----------------------------------------------------------------
# (variant, C, map dtype, out channels-last, z, add_ref, n_src)
GUARDED = {
    "pipe_unstage_nchw": ("pipe", 64, torch.float32, False, False, True, 0),
    "pipe_direct_would_be_cl": ("pipe", 64, torch.bfloat16, True, False, True, 0),
    "pipe_zgemm_c256": ("pipe", 256, torch.float16, False, True, True, 0),
    "pipe_zfp32_c264": ("pipe", 264, torch.bfloat16, True, True, True, 0),
    "pipe_nsrc3_zgemm": ("pipe", 64, torch.bfloat16, False, True, True, 3),
    "tile": ("tile", 64, torch.float32, False, False, True, 0),
    "sector_cl": ("sector", 64, torch.float16, True, False, False, 0),
    "warp_z": ("warp", 64, torch.bfloat16, False, True, True, 0),
}


def _driver_run(f1, f2, P1, P2, K, out_t, od_code, outs, z, variant, add_ref, S, fill):
    p = fusion_params(f1, f2, out_t, K=K, P1=P1, P2=P2, attn=outs["attn"].t, corr=outs["corr"].t, locs_out=outs["locs"].t,
                      z=z, z_residual=z is not None, add_ref=add_ref, variant=variant, n_src=S if S > 1 else 0)
    p.feat_dtype |= _lib.EPI_OUT_DTYPE(od_code)
    nbytes = workspace_bytes(p)
    ws = poisoned(nbytes, fill)
    launch(p, ws)
    assert (ws[nbytes:] == fill).all(), "the guard behind the workspace was written"


@pytest.mark.parametrize("od", OUT16, ids=OD_IDS)
@pytest.mark.parametrize("case", list(GUARDED))
def test_guarded_outputs_over_poisoned_workspace(case, od):
    variant, C, mdt, out_cl, z, add_ref, S = GUARDED[case]
    N, H, W, K = 2, 15, 17, 16
    feats, P, _ = view_inputs(S + 1 if S > 1 else 2, N, C, H, W, K, seed=13)
    f1, f2 = feats[0].to(mdt), feats[1:].flatten(0, 1).to(mdt).contiguous()
    P1, P2 = P[0].contiguous(), P[1:].flatten(0, 1).contiguous()
    zf = random_z(C, 2) if z else None
    NP = max(S, 1) * N
    mk = lambda: dict(attn=Guarded((NP, K, H, W)), corr=Guarded((NP, H, W, 2)), locs=Guarded((K, NP, H, W, 2)))
    ref_outs = mk()
    ref = Guarded((NP, C, H, W), channels_last=out_cl)
    _driver_run(f1, f2, P1, P2, K, ref.t, _lib.EPI_DTYPE_F32, ref_outs, zf, variant, add_ref, S, 0x00)
    runs = []
    for fill in (0x00, 0xFF):
        outs = mk()
        o = Guarded((NP, C, H, W), od, channels_last=out_cl)
        _driver_run(f1, f2, P1, P2, K, o.t, epimod.FEAT_DTYPES[od], outs, zf, variant, add_ref, S, fill)
        o.check("out (workspace 0x%02X)" % fill)
        for k, g in outs.items():
            g.check("%s (workspace 0x%02X)" % (k, fill))
            assert torch.equal(bits(g.t), bits(ref_outs[k].t)), "%s differs from the float32 call" % k
        assert torch.equal(bits(o.t), bits(ref.t.to(od))), "out differs from the float32 out rounded"
        runs.append(o.t.clone())
    assert torch.equal(bits(runs[0]), bits(runs[1])), "out depends on the workspace's old contents"


# ---- 5. the module cast to 16 bits ------------------------------------------------------------------------------------------
def module_cfg(C, H, W, K, z=True):
    return epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                        EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True, PARAMETERIZED=("z",) if z else (), ZRESIDUAL=z),
                        VIS=dict(EPIPOLAR_LINE=True))


def seeded_module(cfg, seed=0):
    m = epi.Epipolar(cfg=cfg).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        C = m.z.weight.shape[0]
        m.z.weight.copy_(torch.randn(m.z.weight.shape, device="cuda", generator=g) / np.sqrt(C))
        m.z.bias.copy_(0.1 * torch.randn(C, device="cuda", generator=g))
        m.bn.weight.copy_(1 + 0.2 * torch.randn(C, device="cuda", generator=g))
        m.bn.bias.copy_(0.1 * torch.randn(C, device="cuda", generator=g))
        m.bn.running_mean.copy_(0.1 * torch.randn(C, device="cuda", generator=g))
        m.bn.running_var.copy_(0.5 + torch.rand(C, device="cuda", generator=g, dtype=torch.float32))
    return m


def upcast_twin(m16, cfg):
    """a float32 module holding the exact float32 values of m16's parameters and buffers"""
    m32 = epi.Epipolar(cfg=cfg).cuda()
    m32.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in m16.state_dict().items()})
    return m32


@pytest.mark.parametrize("cast", ["to_bf16", "half"])
@pytest.mark.parametrize("C", [256, 264], ids=["c256_zgemm", "c264_zfp32"])
def test_cast_module_eval_equals_fp32_rounded(cast, C):
    cfg = module_cfg(C, 16, 20, 16)
    m = seeded_module(cfg)
    m16 = (m.to(torch.bfloat16) if cast == "to_bf16" else m.half()).eval()
    od = torch.bfloat16 if cast == "to_bf16" else torch.float16
    assert m16.out_dtype == od
    m32 = upcast_twin(m16, cfg).eval()
    feats, P, _ = view_inputs(V, 2, C, 16, 20, 16, seed=21)
    feats = feats.to(od)                                          # the backbone of a cast model gives maps of its dtype
    with torch.no_grad():
        for run in (lambda mm: mm(feats[0], feats[1], P[0], P[1]),
                    lambda mm: mm.forward_multi(feats[0], feats[1:4], P[0], P[1:4]),
                    lambda mm: mm.forward_views(feats, P),
                    lambda mm: mm.forward_views(feats, P, sources=TABLE)):
            want = [None if t is None else t.clone() for t in run(m32)]
            got = run(m16)
            torch.cuda.synchronize()
            assert_rounded(got, want, od)


@pytest.mark.parametrize("dtype", OUT16, ids=["bf16", "f16"])
def test_fold_of_16bit_parameters_equals_fold_of_upcast(dtype):
    cfg = module_cfg(256, 16, 16, 16)
    m16 = seeded_module(cfg, seed=4).to(dtype)
    m32 = upcast_twin(m16, cfg)
    wf16, bf16 = epi.fold_z_bn(m16.z, m16.bn)
    wf32, bf32 = epi.fold_z_bn(m32.z, m32.bn)
    torch.cuda.synchronize()
    assert wf16.dtype == torch.float32 and torch.equal(bits(wf16), bits(wf32)) and torch.equal(bits(bf16), bits(bf32))


@pytest.fixture
def deterministic():
    keep = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(keep[0], warn_only=keep[1])


def test_bf16_module_training_step(monkeypatch, deterministic):
    """A training step of a bf16 z + ZRESIDUAL module through `forward` and `forward_views_train`: the fused feature comes back
    in bf16, z / BN / the residual run in bf16 and reach their parameters, and the map gradients are, bit for bit, what the
    float32 layer's backward gives for the same gradient of the fused feature upcast to float32."""
    C, H, W, K = 64, 15, 17, 16
    cfg = module_cfg(C, H, W, K)
    m16 = seeded_module(cfg, seed=6).to(torch.bfloat16).train()
    m32 = epi.Epipolar(cfg=module_cfg(C, H, W, K, z=False)).cuda().train()        # the fused attention alone, in float32
    feats, P, _ = view_inputs(V, 2, C, H, W, K, seed=23)
    feats = feats.to(torch.bfloat16)
    seen = {}
    for name in ("epipolar_fusion_backward", "epipolar_fusion_views_backward"):
        orig = getattr(epimod, name)

        def rec(*a, _orig=orig, _name=name, **kw):
            seen[_name] = a[3 if _name == "epipolar_fusion_views_backward" else 5].detach().clone()   # grad_out as received
            return _orig(*a, **kw)
        monkeypatch.setattr(epimod, name, rec)

    # forward: one (reference, source) pair
    f1, f2 = feats[0].clone().requires_grad_(), feats[1].clone().requires_grad_()
    out, _, attn, _ = m16(f1, f2, P[0], P[1])
    assert out.dtype == torch.bfloat16
    (out.float() * torch.randn_like(out, dtype=torch.float32)).sum().backward()
    g_out = seen["epipolar_fusion_backward"]
    assert g_out.dtype == torch.bfloat16
    assert m16.z.weight.grad is not None and m16.z.weight.grad.dtype == torch.bfloat16 and m16.bn.weight.grad is not None
    r1, r2 = feats[0].clone().requires_grad_(), feats[1].clone().requires_grad_()
    out32, _, _, _ = m32(r1, r2, P[0], P[1])
    assert out32.dtype == torch.float32
    out32.backward(g_out.float())
    assert torch.equal(bits(f1.grad), bits(r1.grad)) and torch.equal(bits(f2.grad), bits(r2.grad))

    # forward_views_train: every view with its table source, from one pass
    fv = feats.clone().requires_grad_()
    outv, _, _, _ = m16.forward_views_train(fv, P, sources=TABLE)
    assert outv.dtype == torch.bfloat16
    (outv.float() * torch.randn_like(outv, dtype=torch.float32)).sum().backward()
    g_v = seen["epipolar_fusion_views_backward"]
    assert g_v.dtype == torch.bfloat16
    rv = feats.clone().requires_grad_()
    out32v, _, _, _ = m32.forward_views_train(rv, P, sources=TABLE)
    out32v.backward(g_v.float().view_as(out32v))
    assert torch.equal(bits(fv.grad), bits(rv.grad))
