"""GPU: the deterministic backward (EpiFusionBwdParams.deterministic, torch.use_deterministic_algorithms).  dL/dfeat_src is
summed in per-pair int64 fixed point, so the same inputs give the same bits: across two runs, inside any batch, for either
layout of the maps and of grad_out.  Checked against the fp64 restatement at the default backward's tolerance, for exact
power-of-two homogeneity, for bf16 / fp16 maps against the fp32 gradient of their values, and for the NaN-pair and
all-far-pair rules.  Each case calls the backward twice on identical inputs; the fp64 references run with the flag off,
because grid_sample's CUDA backward raises under it."""
import contextlib

import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward
from tests.test_gpu_backward import BWD_CASES, BWD_PARAMS, LAYOUT_MODES, LAYOUT_SHAPES, SCALE, TOL, dev, reference_grads, synthetic_pair
from tests.util import edge_locs, rel_max

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def deterministic_algorithms(on=True, warn_only=False):
    """torch.use_deterministic_algorithms for the block, restored afterwards."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.fixture
def det_flag():
    with deterministic_algorithms(True):
        yield


def launches():
    return _lib.load().epi_last_launch_count()


def forward(t1, t2, P1, P2, K, **geo):
    geo.setdefault("softmax_scale", SCALE)
    out, _, attn, locs = epi.epipolar_fusion(t1, t2, P1, P2, K=K, want_locs=True, **geo)
    return out, attn, locs


def grads(seed, out, attn):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(out.shape, device="cuda", generator=g),
            0.3 * torch.randn(attn.shape, device="cuda", generator=g))


@pytest.mark.parametrize("case,other_grad", BWD_PARAMS)
def test_envelope_two_runs_equal_and_fp64(case, other_grad, det_flag):
    """Under the flag (deterministic=None reads it) two runs give equal bits, dL/dfeat_ref is the default path's, both
    gradients match fp64 at 1e-4 of max|grad|, and each path launches its own kernel count."""
    N, C, H, W, K, krt_seed = BWD_CASES[case]
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, krt_seed)
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=krt_seed is None)
    out, attn, locs = forward(t1, t2, P1, P2, **kw)
    g_out, g_attn = grads(3, out, attn)
    bk = dict(grad_attn=g_attn, sample_locs_in=locs, grad_keys="other1" in other_grad, grad_vals="other2" in other_grad, **kw)
    a1, a2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, **bk)
    assert launches() == 5              # staging, coefficient pass, fixed-point scatter, conversion, transposition
    b1, b2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, **bk)
    assert torch.equal(a1, b1) and torch.equal(a2, b2)
    d1, _ = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, deterministic=False, **bk)
    assert launches() == 3              # staging, backward kernel, transposition
    assert torch.equal(a1, d1)
    with deterministic_algorithms(False):
        _, e1, e2 = reference_grads(t1, t2, locs, g_out, g_attn, bk["grad_keys"], bk["grad_vals"])
    assert rel_max(a1.cpu().numpy(), e1.cpu().numpy()) < TOL
    assert rel_max(a2.cpu().numpy(), e2.cpu().numpy()) < TOL


@pytest.mark.parametrize("mode", LAYOUT_MODES)
@pytest.mark.parametrize("shape", LAYOUT_SHAPES)
def test_layouts_and_edges(shape, mode):
    """The layout and edge modes of the default backward's test on the deterministic path: fp64 parity, two equal runs, and
    for the channels_last cases the same bits as the NCHW call, compared after .contiguous()."""
    N, C, H, W, K = shape
    geo = dict(downsample=4.0, img_scale=1.0, align_corners=mode == "align_corners",
               correct_normalize=mode in ("channels_last", "grad_out_stride0", "need_src", "ds8_img_scale"))
    if mode == "ds8_img_scale":
        geo.update(downsample=8.0, img_scale=1.5)
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None, geo["img_scale"], geo["downsample"])
    t1[:, :, 5] = 0.0
    n1, n2 = t1, t2
    if mode == "channels_last":
        t1, t2 = t1.contiguous(memory_format=torch.channels_last), t2.contiguous(memory_format=torch.channels_last)
    locs_in = dev(edge_locs(K, N, H, W, 11)) if mode == "locs_in_edges" else None
    kw = dict(K=K, softmax_scale=SCALE, sample_locs_in=locs_in, **geo)
    out, _, attn, locs = epi.epipolar_fusion(t1, t2, P1, P2, want_locs=True, **kw)
    if mode == "grad_out_stride0":
        g_out, g_attn = torch.ones((1, 1, 1, 1), device="cuda").expand(N, C, H, W), None
    else:
        g_out, g_attn = grads(7, out, attn)
        if mode == "grad_out_channels_last":
            g_out = g_out.contiguous(memory_format=torch.channels_last)
    need_ref, need_src = mode != "need_src", mode != "need_ref"
    bk = dict(grad_attn=g_attn, need_ref=need_ref, need_src=need_src, deterministic=True, **kw)
    g1, g2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, **bk)
    if mode in ("channels_last", "grad_out_channels_last"):     # the second run: the other layout
        h1, h2 = epipolar_fusion_backward(n1, n2, P1, P2, attn, g_out.contiguous(), **bk)
    else:
        h1, h2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, **bk)
    for g, h, t, need in ((g1, h1, t1, need_ref), (g2, h2, t2, need_src)):
        if not need:
            assert g is None and h is None
            continue
        assert g.stride() == t.stride()
        assert torch.equal(g.contiguous(), h.contiguous())
    ro, e1, e2 = reference_grads(t1, t2, locs, g_out, g_attn, align_corners=geo["align_corners"])
    for g, e, need in ((g1, e1, need_ref), (g2, e2, need_src)):
        if need:
            assert rel_max(g.cpu().numpy(), e.cpu().numpy()) < TOL


@pytest.mark.parametrize("use_locs", [True, False], ids=["locs_in", "cameras"])
def test_batch_slices_and_permutation(use_locs):
    """A pair's gradients are the same bits alone, inside the batch and inside a permuted batch: every scale and every sum is
    per pair."""
    N, C, H, W, K = 4, 64, 16, 20, 40
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None)
    out, attn, locs = forward(t1, t2, P1, P2, K, correct_normalize=True)
    g_out, g_attn = grads(5, out, attn)
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=True, deterministic=True)

    def bwd(idx):
        li = locs[:, idx] if use_locs else None
        return epipolar_fusion_backward(t1[idx], t2[idx], P1[idx], P2[idx], attn[idx], g_out[idx], grad_attn=g_attn[idx],
                                        sample_locs_in=li, **kw)

    g1, g2 = bwd(torch.arange(N, device="cuda"))
    perm = torch.tensor([2, 0, 3, 1], device="cuda")
    p1, p2 = bwd(perm)
    assert torch.equal(p1, g1[perm]) and torch.equal(p2, g2[perm])
    s1, s2 = bwd(torch.tensor([1, 2], device="cuda"))
    assert torch.equal(s1, g1[1:3]) and torch.equal(s2, g2[1:3])


@pytest.mark.parametrize("e", [30, -30])
def test_power_of_two_homogeneity(e):
    """Scaling grad_out and grad_attn by 2^e scales both gradients by exactly 2^e: every fp32 step is exact under the
    scaling and the fixed-point scale follows the pair's bound."""
    N, C, H, W, K = 2, 132, 16, 16, 64
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, 2)
    out, attn, locs = forward(t1, t2, P1, P2, K)
    g_out, g_attn = grads(9, out, attn)
    kw = dict(K=K, softmax_scale=SCALE, sample_locs_in=locs, deterministic=True)
    g1, g2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, grad_attn=g_attn, **kw)
    f = 2.0 ** e
    s1, s2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out * f, grad_attn=g_attn * f, **kw)
    assert torch.equal(s1, g1 * f) and torch.equal(s2, g2 * f)
    assert g2.abs().max() > 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("C", [64, 17])
def test_lowp_maps_exact(dtype, C):
    """bf16 / fp16 maps give exactly the deterministic fp32 gradient of their float values, rounded once to the map's dtype."""
    N, H, W, K = 2, 12, 20, 40
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None)
    l1, l2 = t1.to(dtype), t2.to(dtype)
    out, attn, locs = forward(l1, l2, P1, P2, K, correct_normalize=True)
    g_out, g_attn = grads(11, out, attn)
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=True, grad_attn=g_attn, sample_locs_in=locs, deterministic=True)
    g1, g2 = epipolar_fusion_backward(l1, l2, P1, P2, attn, g_out, **kw)
    assert launches() == 7              # + the reference conversion and its gradient's transposition
    f1, f2 = epipolar_fusion_backward(l1.float(), l2.float(), P1, P2, attn, g_out, **kw)
    assert g1.dtype == dtype and g2.dtype == dtype
    assert torch.equal(g1, f1.to(dtype)) and torch.equal(g2, f2.to(dtype))


def test_nan_pair_and_far_pair():
    """A NaN in one pair's grad_out makes that pair's dL/dfeat_src all NaN and leaves the other pairs' bits alone; a pair whose
    samples all lie far off the map gets zeros."""
    N, C, H, W, K = 3, 64, 12, 16, 32
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None)
    out, attn, locs = forward(t1, t2, P1, P2, K, correct_normalize=True)
    locs = locs.clone()
    locs[:, 2] = 10000.0                                       # pair 2: no sample has a tap
    g_out, g_attn = grads(13, out, attn)
    y, x = 6, 8
    assert (locs[:, 1, y, x].abs() < 1).all(-1).any()          # pixel (6, 8) of pair 1 has samples on the map
    bad = g_out.clone()
    bad[1, 3, y, x] = float("nan")
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=True, grad_attn=g_attn, sample_locs_in=locs, deterministic=True)
    g1, g2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, g_out, **kw)
    n1, n2 = epipolar_fusion_backward(t1, t2, P1, P2, attn, bad, **kw)
    assert torch.isnan(n2[1]).all()
    assert torch.equal(n2[0], g2[0]) and torch.equal(n2[2], g2[2])
    assert torch.equal(g2[2], torch.zeros_like(g2[2])) and torch.equal(g1[2], torch.zeros_like(g1[2]))
    assert g2[0].abs().max() > 0


def test_module_train_steps_equal(det_flag):
    """`Epipolar` in train mode under torch.use_deterministic_algorithms(True): two identical steps give equal gradients, and
    they are the deterministic path's (autograd runs the backward on its own thread, so the launch count of this thread does
    not show the path; the bits do)."""
    N, C, H, W, K = 2, 64, 16, 16, 32
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True),
                       VIS=dict(EPIPOLAR_LINE=True))
    m = epi.Epipolar(cfg=cfg).cuda().train()
    t1, t2, P1, P2 = synthetic_pair(N, C, H, W, K, None)
    gen = torch.Generator(device="cuda").manual_seed(17)
    w, w_attn = torch.randn((N, C, H, W), device="cuda", generator=gen), torch.randn((N, K, H, W), device="cuda", generator=gen)
    got = []
    for _ in range(2):
        a, b = t1.clone().requires_grad_(True), t2.clone().requires_grad_(True)
        out, corr, attn, locs = m(a, b, P1, P2)
        ((out * w).sum() + (attn * w_attn).sum()).backward()
        got.append((a.grad, b.grad))
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    assert got[0][1].abs().max() > 0
    d1, d2 = epipolar_fusion_backward(t1, t2, P1, P2, attn.detach(), w, K=K, softmax_scale=SCALE, correct_normalize=True,
                                      grad_attn=w_attn, sample_locs_in=locs.transpose(0, 1), deterministic=True)
    assert torch.equal(got[0][0], d1) and torch.equal(got[0][1], d2)
