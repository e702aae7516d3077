"""GPU: backward of the fused attention (SURVEY.md 8f rank 1) against PyTorch autograd through the reference's own op
composition (F.grid_sample x2, mul/sum, ==0 mask assignment, softmax, weighted sum — epipolar.py:188-247) evaluated in
float64 on the same sample locations.  Tolerance 1e-4 relative to max|grad| (fp32 kernel, float atomics)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.epipolar import _FusionFn, epipolar_fusion_backward
from oracle import golden_cases as gc
from tests.util import edge_locs, rel_max

pytestmark = pytest.mark.gpu
TOL = 1e-4
SCALE = float(epi.make_cfg().EPIPOLAR.SOFTMAXSCALE)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def torch_reference(f1, f2k, f2v, locs, scale, align_corners=False):
    """differentiable restatement in the dtype of the inputs; f2k / f2v = the source map as 'other1' / 'other2'.
    f1 [N,C,h,w] and locs [K,N,h,w,2] may be a band of reference rows; the source maps are always whole.  grid_sample samples
    every grid point on its own, so the K sample grids are stacked along the grid's rows: the same numbers as sampling a
    K-fold expanded source map, without the K·C·H·W input gradient that expansion costs in the backward."""
    N, C, h, w = f1.shape
    K = locs.shape[0]
    outs, attns = [], []
    for n in range(N):
        g = locs[:, n].reshape(1, K * h, w, 2)
        keys = F.grid_sample(f2k[n:n + 1], g, align_corners=align_corners).view(C, K, h, w).transpose(0, 1)
        vals = F.grid_sample(f2v[n:n + 1], g, align_corners=align_corners).view(C, K, h, w).transpose(0, 1)
        sim = (keys * f1[n].unsqueeze(0)).sum(1)
        sim = torch.where(sim == 0, torch.full_like(sim, -1e10), sim)          # `sim[sim==0] = -1e10`: no gradient there
        a = F.softmax(sim * scale, 0)
        outs.append((vals * a.unsqueeze(1)).sum(0))
        attns.append(a)
    return torch.stack(outs), torch.stack(attns)


def reference_grads(f1, f2, locs, g_out, g_attn, grad_keys=True, grad_vals=True, align_corners=False, budget=1 << 23):
    """fp64 (out, dL/dfeat_ref, dL/dfeat_src) of  L = Σ out·g_out + Σ attn·g_attn  (g_attn may be None) through
    torch_reference on the given sample locations.  Evaluated over bands of reference rows whose gradients add up, so that
    no K·C·rows·W intermediate holds more than `budget` elements (64 MB in fp64)."""
    N, C, H, W = f1.shape
    K = locs.shape[0]
    r1 = f1.detach().double().requires_grad_(True)
    r2 = f2.detach().double().requires_grad_(True)
    r2k = r2 if grad_keys else r2.detach()
    r2v = r2 if grad_vals else r2.detach()
    locs = locs.double()
    rows = max(1, min(H, budget // (K * C * W)))
    out = torch.empty_like(r1, requires_grad=False)
    e1, e2 = torch.zeros_like(out), torch.zeros_like(out)
    for y0 in range(0, H, rows):
        band = slice(y0, y0 + rows)
        ro, ra = torch_reference(r1[:, :, band], r2k, r2v, locs[:, :, band], SCALE, align_corners)
        loss = (ro * g_out[:, :, band].double()).sum()
        if g_attn is not None:
            loss = loss + (ra * g_attn[:, :, band].double()).sum()
        d1, d2 = torch.autograd.grad(loss, (r1, r2), allow_unused=True)
        e1 += d1
        if d2 is not None:
            e2 += d2
        out[:, :, band] = ro.detach()
    return out, e1, e2


def synthetic_pair(N, C, H, W, K, krt_seed, img_scale=1.0, downsample=4.0):
    """randn features; ring cameras (krt_seed None) or literal randn KRTs, whose lines miss the map for some pixels."""
    if krt_seed is None:
        P1, P2 = syn.pairs_from_ring(max(N, 2), int(max(H, W) * downsample * img_scale), seed=K)
        P1, P2 = P1[:N], P2[:N]
    else:
        P1, P2 = syn.random_krt(N, seed=krt_seed)
    f1, f2 = syn.features(N, C, H, W, "randn", 5), syn.features(N, C, H, W, "randn", 6)
    return dev(f1), dev(f2), dev(P1.astype(np.float32)), dev(P2.astype(np.float32))


@pytest.mark.parametrize("name", ["tiny_ring_z", "tiny_randn_krt", "tiny_zero_query", "cfg1_ring"])
@pytest.mark.parametrize("other_grad", [("other1", "other2"), ("other2",), ("other1",)])
def test_backward_vs_autograd_fp64(name, other_grad):
    cfg, f1, f2, P1, P2, _ = gc.build_inputs(name)
    spec = gc.CASES[name]
    if name == "cfg1_ring" and other_grad != ("other1", "other2"):
        pytest.skip("one OTHER_GRAD setting is enough at this size")
    K = spec["K"]
    t1 = dev(f1).requires_grad_(True); t2 = dev(f2).requires_grad_(True)
    opts = dict(fwd=dict(K=K, downsample=cfg.BACKBONE.DOWNSAMPLE, img_scale=cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE,
                         softmax_scale=cfg.EPIPOLAR.SOFTMAXSCALE, correct_normalize=spec["correct"], align_corners=False,
                         want_corr=True, want_locs=True, variant="auto"),
                grad_keys="other1" in other_grad, grad_vals="other2" in other_grad)
    out, corr, attn, locs = _FusionFn.apply(t1, t2, dev(P1), dev(P2), opts)
    torch.manual_seed(3)
    w_out = torch.randn_like(out); w_attn = torch.randn_like(attn)
    loss = (out * w_out).sum() + 0.3 * (attn * w_attn).sum()                    # a loss that also touches the attention output
    g1, g2 = torch.autograd.grad(loss, (t1, t2))
    # reference in float64 on the locations the kernel sampled
    r1 = dev(f1).double().requires_grad_(True); r2 = dev(f2).double().requires_grad_(True)
    r2k = r2 if "other1" in other_grad else r2.detach()
    r2v = r2 if "other2" in other_grad else r2.detach()
    ro, ra = torch_reference(r1, r2k, r2v, locs.double(), float(cfg.EPIPOLAR.SOFTMAXSCALE))
    rloss = (ro * w_out.double()).sum() + 0.3 * (ra * w_attn.double()).sum()
    e1, e2 = torch.autograd.grad(rloss, (r1, r2), allow_unused=True)
    assert rel_max(out.detach().cpu().numpy(), ro.detach().cpu().numpy()) < 1e-4
    assert rel_max(g1.cpu().numpy(), e1.cpu().numpy()) < 1e-4
    assert rel_max(g2.cpu().numpy(), e2.cpu().numpy()) < 1e-4


def test_module_trains_end_to_end():
    """Epipolar under autograd in train mode (engine/trainer.py:72): gradients reach both feature maps and z / bn, and
    match the PyTorch composition (conv1x1 + BatchNorm(train) + ZRESIDUAL on top of the reference attention)."""
    name = "tiny_ring_z"
    cfg, f1, f2, P1, P2, params = gc.build_inputs(name)
    cfg.VIS.EPIPOLAR_LINE = True
    torch.backends.cudnn.allow_tf32 = False            # the module's own conv1x1 (PyTorch) must not run in TF32 for a 1e-4 comparison
    torch.backends.cuda.matmul.allow_tf32 = False
    m = epi.Epipolar(cfg=cfg).cuda().train()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    t1 = dev(f1).requires_grad_(True); t2 = dev(f2).requires_grad_(True)
    out, corr, attn, locs_t = m(t1, t2, dev(P1), dev(P2))
    w = torch.randn_like(out)
    (out * w).sum().backward()
    assert t1.grad is not None and t2.grad is not None and m.z.weight.grad is not None and m.bn.weight.grad is not None
    # reference composition in float64
    mz = torch.nn.Conv2d(m.z.in_channels, m.z.out_channels, 1).cuda().double()
    mz.load_state_dict({k: v.double() for k, v in m.z.state_dict().items()})
    r1 = dev(f1).double().requires_grad_(True); r2 = dev(f2).double().requires_grad_(True)
    locs = locs_t.transpose(0, 1).contiguous().double()
    ro, _ = torch_reference(r1, r2, r2, locs, float(cfg.EPIPOLAR.SOFTMAXSCALE))
    y = F.batch_norm(mz(ro), None, None, m.bn.weight.double(), m.bn.bias.double(), True, 0.1, m.bn.eps) + ro
    (y * w.double()).sum().backward()
    assert rel_max(out.detach().cpu().numpy(), y.detach().cpu().numpy()) < 1e-4
    assert rel_max(t1.grad.cpu().numpy(), r1.grad.cpu().numpy()) < 2e-4
    assert rel_max(t2.grad.cpu().numpy(), r2.grad.cpu().numpy()) < 2e-4
    assert rel_max(m.z.weight.grad.cpu().numpy(), mz.weight.grad.cpu().numpy()) < 2e-4


# (N, C, H, W, K, random-KRT seed or None for ring cameras): every instantiation of the backward kernel at the ends of its
# channel range, K from the two endpoints alone up to eight 32-sample chunks, and the full training shape
BWD_CASES = {
    "c4_k2": (2, 4, 12, 16, 2, None),                  # <4,1>, endpoints only
    "c3_k33": (1, 3, 16, 16, 33, 0),                   # <1,1>, a partial second chunk
    "c31_k64": (2, 31, 12, 20, 64, None),              # <1,1> at its largest C, two full chunks
    "c33_k65": (1, 33, 16, 16, 65, 0),                 # <1,4> at its smallest C, three chunks
    "c126_k32": (1, 126, 16, 16, 32, None),            # <1,4> at its largest C (C % 4 == 2)
    "c128_k96": (2, 128, 16, 16, 96, 2),               # <4,1> at its largest C
    "c132_k64": (1, 132, 16, 16, 64, None),            # <4,2> at its smallest C
    "c256_k64": (2, 256, 32, 32, 64, 2),               # <4,2>, the production C and K
    "c260_k128": (1, 260, 16, 16, 128, None),          # <4,4> at its smallest C
    "c512_k256": (1, 512, 12, 16, 256, 0),             # <4,4> at its largest C, K = 256 (eight chunks)
    "train_c256_k64_64x64": (1, 256, 64, 64, 64, None),   # training shape: the fp64 reference runs in bands of rows
}
BOTH = ("other1", "other2")
BWD_PARAMS = [pytest.param(name, BOTH, id=name + "-both") for name in BWD_CASES] + [
    pytest.param(name, og, id="%s-%s" % (name, og[0])) for name in ("c33_k65", "c256_k64") for og in (("other1",), ("other2",))]


@pytest.mark.parametrize("case,other_grad", BWD_PARAMS)
def test_backward_envelope_vs_autograd_fp64(case, other_grad):
    """The backward across its instantiations and sample chunks, under autograd as training runs it: out, dL/dfeat_ref and
    dL/dfeat_src against the fp64 restatement on the locations the forward emitted.  The random KRTs leave whole pixels on
    the far sentinel (no taps, every sample masked)."""
    N, C, H, W, K, krt_seed = BWD_CASES[case]
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, krt_seed)
    t1.requires_grad_(True); t2.requires_grad_(True)
    grad_keys, grad_vals = "other1" in other_grad, "other2" in other_grad
    opts = dict(fwd=dict(K=K, downsample=4.0, img_scale=1.0, softmax_scale=SCALE, correct_normalize=krt_seed is None,
                         align_corners=False, want_corr=True, want_locs=True, variant="auto"),
                grad_keys=grad_keys, grad_vals=grad_vals)
    out, _, attn, locs = _FusionFn.apply(t1, t2, P1, P2, opts)
    if krt_seed is not None:
        far = (locs.abs() >= 50).all(-1).all(0)                                  # [N,H,W]: the line misses the source map
        assert 0 < far.float().mean().item() < 1
    torch.manual_seed(3)
    w_out, w_attn = torch.randn_like(out), torch.randn_like(attn)
    loss = (out * w_out).sum() + 0.3 * (attn * w_attn).sum()
    g1, g2 = torch.autograd.grad(loss, (t1, t2))
    ro, e1, e2 = reference_grads(t1, t2, locs, w_out, 0.3 * w_attn, grad_keys, grad_vals)
    assert rel_max(out.detach().cpu().numpy(), ro.cpu().numpy()) < TOL
    assert rel_max(g1.cpu().numpy(), e1.cpu().numpy()) < TOL
    assert rel_max(g2.cpu().numpy(), e2.cpu().numpy()) < TOL


LAYOUT_SHAPES = [pytest.param((2, 64, 12, 20, 48), id="vec4_c64_k48"), pytest.param((2, 17, 12, 20, 40), id="vec1_c17_k40")]
LAYOUT_MODES = ["channels_last", "grad_out_channels_last", "grad_out_stride0", "align_corners", "ds8_img_scale",
                "need_ref", "need_src", "locs_in_edges"]


@pytest.mark.parametrize("mode", LAYOUT_MODES)
@pytest.mark.parametrize("shape", LAYOUT_SHAPES)
def test_backward_layouts_and_edges(shape, mode):
    """`epipolar_fusion_backward` with the caller's layouts (channels_last maps, a channels_last grad_out, the stride-0
    grad_out autograd passes for loss = out.sum()), the geometry options, one-sided gradients and injected edge-case
    locations, vs the fp64 restatement.  Query row 5 is all zero: every sample masked, uniform attention.  Without injected
    locations the backward derives them from the (well-conditioned ring) cameras itself."""
    N, C, H, W, K = shape
    geo = dict(downsample=4.0, img_scale=1.0, align_corners=mode == "align_corners",
               correct_normalize=mode in ("channels_last", "grad_out_stride0", "need_src", "ds8_img_scale"))
    if mode == "ds8_img_scale":
        geo.update(downsample=8.0, img_scale=1.5)
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None, geo["img_scale"], geo["downsample"])
    t1[:, :, 5] = 0.0
    if mode == "channels_last":
        t1, t2 = t1.contiguous(memory_format=torch.channels_last), t2.contiguous(memory_format=torch.channels_last)
    locs_in = dev(edge_locs(K, N, H, W, 11)) if mode == "locs_in_edges" else None
    kw = dict(K=K, softmax_scale=SCALE, sample_locs_in=locs_in, **geo)
    out, _, attn, locs = epi.epipolar_fusion(t1, t2, P1, P2, want_locs=True, **kw)
    if locs_in is not None:
        assert torch.equal(locs, locs_in)
    torch.manual_seed(7)
    if mode == "grad_out_stride0":
        g_out, g_attn = torch.ones((1, 1, 1, 1), device="cuda").expand(N, C, H, W), None
        assert g_out.stride() == (0, 0, 0, 0)
    else:
        g_out, g_attn = torch.randn_like(out), torch.randn_like(attn)
        if mode == "grad_out_channels_last":
            g_out = g_out.contiguous(memory_format=torch.channels_last)
    need_ref, need_src = mode != "need_src", mode != "need_ref"
    g1, g2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, grad_attn=g_attn, need_ref=need_ref, need_src=need_src, **kw)
    ro, e1, e2 = reference_grads(t1, t2, locs, g_out, g_attn, align_corners=geo["align_corners"])
    assert rel_max(out.cpu().numpy(), ro.cpu().numpy()) < TOL
    for g, e, t, need in ((g1, e1, t1, need_ref), (g2, e2, t2, need_src)):
        if not need:
            assert g is None
            continue
        assert g.stride() == t.stride()
        assert rel_max(g.cpu().numpy(), e.cpu().numpy()) < TOL
