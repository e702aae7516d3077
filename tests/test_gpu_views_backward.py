"""GPU: the backward of the views form (`epipolar_fusion_views_backward`, `Epipolar.forward_views_train`).  Each view item's
gradient is the sum, over the pairs it is the query of, of dL/dfeat_ref and, over the pairs that name it as their source, of
dL/dfeat_src; every term is checked against fp64 autograd through the reference's op composition on the locations the forward
sampled.  The query terms alone (S = 1, OTHER_GRAD empty) must be the one-pair backward's bits, the deterministic path must
not depend on the batch around a frame or the layout, and a training step from one backbone pass must match the reference's
two-pass step (modeling/model.py:240-247)."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward
from tests.test_gpu_backward import SCALE, TOL, reference_grads
from tests.test_gpu_buffers import Guarded, int_bits, poisoned
from tests.test_gpu_view_sources import TABLES, table
from tests.test_gpu_views import DT_IDS, DTYPES, others, view_inputs
from tests.util import bwd_params, rel_max

pytestmark = pytest.mark.gpu
OTHER_GRADS = {"both": ("other1", "other2"), "other1": ("other1",), "other2": ("other2",), "none": ()}
PATHS = [False, True]
PATH_IDS = ["default", "det"]


def rows(kind, V):
    """the [V,S] source rows of a table kind, or every other view (kind None)"""
    return [others(V, v) for v in range(V)] if kind is None else table(kind, V)


def lowp_tol(dtype):
    return TOL + (torch.finfo(dtype).eps if dtype != torch.float32 else 0.0)


def inputs(V, N, C, H, W, K, seed):
    """view_inputs without the K keyword: feats [V,N,C,H,W], P [V,N,3,4], geometry kwargs"""
    feats, P, kw = view_inputs(V, N, C, H, W, K, seed=seed)
    kw.pop("K")
    return feats, P, kw


def run_forward(feats, P, kind, K, **kw):
    """the views forward -> (attn [V,S,N,K,H,W], locs [K,V,S,N,H,W,2], source rows, sources argument)"""
    V = feats.shape[0]
    src = rows(kind, V)
    sources = None if kind is None else src
    _, _, attn, locs = epi.epipolar_fusion_views(feats, P, K=K, softmax_scale=SCALE, want_locs=True, sources=sources, **kw)
    return attn, locs, src, sources


def loss_weights(attn, C, seed, with_attn=True):
    """dL/dout [V,S,N,C,H,W] and dL/dattn (or None) of  L = Σ out·w_out + 0.3 Σ attn·w_attn"""
    V, S, N, K, H, W = attn.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    w_out = torch.randn((V, S, N, C, H, W), device="cuda", generator=g)
    w_attn = 0.3 * torch.randn(attn.shape, device="cuda", generator=g) if with_attn else None
    return w_out, w_attn


def pair_items(src, N):
    """query and source view items of every pair p = (v·S + j)·N + n"""
    q = [v * N + n for v in range(len(src)) for _ in src[v] for n in range(N)]
    u = [s * N + n for v in range(len(src)) for s in src[v] for n in range(N)]
    return torch.tensor(q, device="cuda"), torch.tensor(u, device="cuda")


def fp64_grads(feats, locs, w_out, w_attn, src, grad_keys=True, grad_vals=True, align_corners=False):
    """fp64 dL/dfeats [V,N,C,H,W]: each pair's dL/dfeat_ref and dL/dfeat_src (reference_grads on the gathered pair batch),
    index_add-ed into the view items"""
    V, N, C, H, W = feats.shape
    q, u = pair_items(src, N)
    f = feats.float().flatten(0, 1)
    NP = q.numel()
    _, e1, e2 = reference_grads(f[q], f[u], locs.flatten(1, 3), w_out.reshape(NP, C, H, W),
                                None if w_attn is None else w_attn.reshape(NP, -1, H, W), grad_keys, grad_vals, align_corners)
    g = torch.zeros((V * N, C, H, W), device="cuda", dtype=torch.float64)
    g.index_add_(0, q, e1)
    g.index_add_(0, u, e2)
    return g.view(V, N, C, H, W)


def views_bwd(feats, attn, w_out, w_attn, locs, sources, K, det, other_grad=("other1", "other2"), **kw):
    return epi.epipolar_fusion_views_backward(feats, None, attn, w_out, K=K, softmax_scale=SCALE, sources=sources,
                                              grad_attn=w_attn, sample_locs_in=locs, grad_keys="other1" in other_grad,
                                              grad_vals="other2" in other_grad, deterministic=det, **kw)


def check_vs_fp64(feats, P, kind, K, det, other_grad=("other1", "other2"), with_attn=True, seed=3, locs_in=None, **kw):
    attn, locs, src, sources = run_forward(feats, P, kind, K, **kw)
    if locs_in is not None:                                    # the forward again, on the injected locations
        attn, locs, src, sources = run_forward(feats, P, kind, K, sample_locs_in=locs_in(locs), **kw)
    w_out, w_attn = loss_weights(attn, feats.shape[2], seed, with_attn)
    g = views_bwd(feats, attn, w_out, w_attn, locs, sources, K, det, other_grad,
                  correct_normalize=kw.get("correct_normalize", False))
    assert g.shape == feats.shape and g.dtype == feats.dtype
    e = fp64_grads(feats, locs, w_out, w_attn, src, "other1" in other_grad, "other2" in other_grad)
    assert e.abs().max().item() > 0
    err = rel_max(g.float().cpu().numpy(), e.cpu().numpy())
    assert err < lowp_tol(feats.dtype), err
    return g


# ---- 1. against fp64 autograd ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("N", [1, 2])
@pytest.mark.parametrize("V", [2, 4, 5])
@pytest.mark.parametrize("kind", TABLES + [None], ids=TABLES + ["all_others"])
def test_tables_vs_fp64(kind, V, N, det):
    if kind == "nobodys_source" and V == 2:
        pytest.skip("with two views each is the other's source")
    feats, P, kw = inputs(V, N, 16, 12, 16, 16, seed=V + N)
    check_vs_fp64(feats, P, kind, 16, det, **kw)


@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("with_attn", [True, False], ids=["grad_attn", "no_grad_attn"])
@pytest.mark.parametrize("other_grad", list(OTHER_GRADS))
def test_other_grad_vs_fp64(other_grad, with_attn, det):
    """OTHER_GRAD selects the source terms: 'none' leaves the query terms alone, as in the reference with the source pass
    under no_grad"""
    feats, P, kw = inputs(4, 2, 32, 12, 16, 24, seed=21)
    check_vs_fp64(feats, P, "s2", 24, det, OTHER_GRADS[other_grad], with_attn, **kw)


@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("dtype", DTYPES[1:], ids=DT_IDS[1:])
def test_lowp_vs_fp64(dtype, det):
    """bf16 / fp16 maps: fp32 sums rounded once, within the one-pair backward's low-precision tolerance"""
    feats, P, kw = inputs(4, 2, 64, 13, 21, 48, seed=8)
    check_vs_fp64(feats.to(dtype), P, "duplicates", 48, det, **kw)


# ---- 2. the query terms are the one-pair backward's bits ------------------------------------------------------------------
@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind", ["nearest", "everybodys_source"])
def test_query_terms_equal_single_backward(kind, dtype, det):
    V, N, K = 4, 2, 32
    feats, P, kw = inputs(V, N, 64, 16, 16, K, seed=5)
    feats = feats.to(dtype)
    attn, locs, src, sources = run_forward(feats, P, kind, K, **kw)
    w_out, w_attn = loss_weights(attn, 64, 6)
    g = views_bwd(feats, attn, w_out, w_attn, locs, sources, K, det, other_grad=(), correct_normalize=True)
    for v in range(V):
        u = src[v][0]
        want, _ = epipolar_fusion_backward(feats[v], feats[u], P[v], P[u], attn[v, 0], w_out[v, 0], K=K, softmax_scale=SCALE,
                                           correct_normalize=True, grad_attn=w_attn[v, 0], sample_locs_in=locs[:, v, 0],
                                           grad_keys=False, grad_vals=False, need_src=False, deterministic=det)
        assert torch.equal(g[v], want), v


# ---- 3. determinism -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_deterministic_runs_frames_and_layouts(dtype):
    """two runs give the same bits; frame n gives the same bits alone (N = 1) as inside an N = 3 batch; NCHW and channels_last
    maps give the same values"""
    V, N, C, K = 4, 3, 64, 32
    feats, P, kw = inputs(V, N, C, 16, 20, K, seed=9)
    feats = feats.to(dtype)
    kind = "duplicates"
    attn, locs, src, sources = run_forward(feats, P, kind, K, **kw)
    w_out, w_attn = loss_weights(attn, C, 10)
    run = lambda f, a, wo, wa, l: views_bwd(f, a, wo, wa, l, sources, K, True, correct_normalize=True)
    g = run(feats, attn, w_out, w_attn, locs)
    assert torch.equal(int_bits(g), int_bits(run(feats, attn, w_out, w_attn, locs)))
    assert g.abs().max() > 0
    for n in range(N):
        s = slice(n, n + 1)
        alone = run(feats[:, s].contiguous(), attn[:, :, s].contiguous(), w_out[:, :, s].contiguous(), w_attn[:, :, s].contiguous(),
                    locs[:, :, :, s].contiguous())
        assert torch.equal(int_bits(alone[:, 0]), int_bits(g[:, n])), n
    cl = feats.flatten(0, 1).contiguous(memory_format=torch.channels_last).unflatten(0, (V, N))
    g_cl = run(cl, attn, w_out, w_attn, locs)
    assert g_cl.flatten(0, 1).is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(g_cl, g)


def test_deterministic_nan_stays_in_its_frame():
    """a NaN in one frame's map makes that frame's source-fed item gradient all NaN (its pair's bound is not finite) and
    leaves every other frame finite"""
    V, N, C, K = 4, 3, 32, 16
    feats, P, kw = inputs(V, N, C, 12, 16, K, seed=13)
    attn, locs, src, sources = run_forward(feats, P, "nearest", K, **kw)
    w_out, w_attn = loss_weights(attn, C, 14)
    bad = feats.clone()
    bad[0, 1, 3, 5, 7] = float("nan")                          # view 0 of frame 1, the query of pair (0, 0, 1)
    g = views_bwd(bad, attn, w_out, w_attn, locs, sources, K, True, correct_normalize=True)
    assert torch.isnan(g[src[0][0], 1]).all()                  # its source item: view 1 of frame 1
    assert torch.isfinite(g[:, 0]).all() and torch.isfinite(g[:, 2]).all()


# ---- 4. shapes: every backward instantiation, odd maps, layouts, injected locations, the training shape ----------------------
SHAPES = {                                    # (V, N, C, H, W, K): C picks the instantiation <VEC, NV>
    "c30_k33_13x17": (4, 2, 30, 13, 17, 33),  # <1,1>
    "c64_k2_12x16": (4, 2, 64, 12, 16, 2),    # <4,1>, the two endpoints alone
    "c66_k64_13x17": (3, 2, 66, 13, 17, 64),  # <1,4>
    "c132_k33_12x12": (3, 1, 132, 12, 12, 33),   # <4,2>
    "c264_k64_10x12": (3, 1, 264, 10, 12, 64),   # <4,4>
}


@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_shapes_vs_fp64(shape, det):
    V, N, C, H, W, K = SHAPES[shape]
    feats, P, kw = inputs(V, N, C, H, W, K, seed=C)
    check_vs_fp64(feats, P, "s2", K, det, **kw)


@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("layout", ["channels_last", "strided", "locs_in"])
def test_layouts_vs_fp64(layout, det):
    """channels_last maps, a channel slice of a wider buffer (a strided view) and perturbed injected locations"""
    V, N, C, H, W, K = 4, 2, 32, 13, 17, 24
    feats, P, kw = inputs(V, N, C, H, W, K, seed=17)
    locs_in = None
    if layout == "channels_last":
        feats = feats.flatten(0, 1).contiguous(memory_format=torch.channels_last).unflatten(0, (V, N))
    elif layout == "strided":
        wide = torch.randn((V, N, C + 5, H, W), device="cuda")
        wide[:, :, 2:2 + C] = feats
        feats = wide[:, :, 2:2 + C]
    else:
        g = torch.Generator(device="cuda").manual_seed(18)
        locs_in = lambda l: (l + 0.03 * (torch.rand(l.shape, device="cuda", generator=g) - 0.5)).contiguous()
    check_vs_fp64(feats, P, "nearest", K, det, locs_in=locs_in, **kw)


def test_training_shape_vs_fp64():
    """V = 4 views, N = 4 frames, the nearest camera (16 pairs), C = 256, 64x64, K = 64: both paths against one fp64 reference"""
    V, N, C, H, W, K = 4, 4, 256, 64, 64, 64
    feats, P, kw = inputs(V, N, C, H, W, K, seed=2)
    attn, locs, src, sources = run_forward(feats, P, "nearest", K, **kw)
    w_out, w_attn = loss_weights(attn, C, 4)
    e = fp64_grads(feats, locs, w_out, w_attn, src).cpu().numpy()
    for det in PATHS:
        g = views_bwd(feats, attn, w_out, w_attn, locs, sources, K, det, correct_normalize=True)
        assert rel_max(g.cpu().numpy(), e) < TOL, det


# ---- 5. the module against the gathered flow ------------------------------------------------------------------------------
def module_cfg(C, H, W, K):
    return epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                        EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True, PARAMETERIZED=("z",), ZRESIDUAL=True),
                        VIS=dict(EPIPOLAR_LINE=True))


@pytest.fixture
def no_tf32():
    keep = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = keep


@pytest.mark.parametrize("fuse_ref", [False, True])
def test_forward_views_train_equals_gathered_forward(fuse_ref, no_tf32):
    """training mode with z + ZRESIDUAL: the outputs equal `forward` on the gathered V·S·N pair batch bit for bit, BatchNorm's
    running statistics after the step too, and the gradients of feats, z and bn agree to 1e-5"""
    V, N, C, H, W, K = 4, 2, 64, 16, 16, 32
    cfg = module_cfg(C, H, W, K)
    m = epi.Epipolar(cfg=cfg, fuse_ref_residual=fuse_ref).cuda().train()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.z_bn_params(C, 5).items()}, strict=False)
    ref = copy.deepcopy(m)
    feats, P, _ = view_inputs(V, N, C, H, W, K, seed=22)
    src = table("s2", V)
    q, u = pair_items(src, N)
    a = feats.clone().requires_grad_(True)
    got = m.forward_views_train(a, P, sources=src)
    b = feats.clone().requires_grad_(True)
    fb, Pf = b.flatten(0, 1), P.flatten(0, 1)
    want = ref(fb[q], fb[u], Pf[q], Pf[u])
    pairs = (V, len(src[0]), N)
    for i, what in enumerate(("finalout", "corr_pos", "attn")):
        assert torch.equal(got[i], want[i].unflatten(0, pairs)), what
    assert torch.equal(got[3], want[3].unflatten(0, pairs)), "sample_locs"
    assert torch.equal(m.bn.running_mean, ref.bn.running_mean) and torch.equal(m.bn.running_var, ref.bn.running_var)
    gen = torch.Generator(device="cuda").manual_seed(23)
    w, w_attn = torch.randn(got[0].shape, device="cuda", generator=gen), torch.randn(got[2].shape, device="cuda", generator=gen)
    ((got[0] * w).sum() + (got[2] * w_attn).sum()).backward()
    ((want[0] * w.flatten(0, 2)).sum() + (want[2] * w_attn.flatten(0, 2)).sum()).backward()
    for what, x, y in (("feats", a.grad, b.grad), ("z.weight", m.z.weight.grad, ref.z.weight.grad),
                       ("z.bias", m.z.bias.grad, ref.z.bias.grad), ("bn.weight", m.bn.weight.grad, ref.bn.weight.grad),
                       ("bn.bias", m.bn.bias.grad, ref.bn.bias.grad)):
        assert rel_max(x.cpu().numpy(), y.cpu().numpy()) < 1e-5, what


# ---- 6. a training step from one backbone pass against the reference's two-pass step -------------------------------------
class Backbone(torch.nn.Module):
    """a stand-in for the pose network's backbone: conv-BN-ReLU twice, to C channels at stride 4 (no conv bias in front of a
    BatchNorm, as in a ResNet: its gradient would be zero up to rounding)"""

    def __init__(self, C):
        super().__init__()
        self.body = torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, 2, 1, bias=False), torch.nn.BatchNorm2d(32), torch.nn.ReLU(),
                                        torch.nn.Conv2d(32, C, 3, 2, 1, bias=False), torch.nn.BatchNorm2d(C), torch.nn.ReLU())

    def forward(self, x):
        return self.body(x)


def test_one_pass_step_equals_two_pass_step(no_tf32):
    """Each of the V·N views is fused with view (v + 1) % V.  The reference runs the shared backbone on `other_img` (the
    permuted views) and then on `img`, and fuses the two batches; here one backbone pass over the views feeds
    `forward_views_train`.  With a permutation table the loss and every parameter gradient agree to 1e-4 (BatchNorm batch
    statistics do not depend on the order; the running statistics are updated once instead of twice, so they are left out)."""
    V, N, C, K, J = 4, 2, 32, 16, 5
    H = W = 16
    cfg = module_cfg(C, H, W, K)
    torch.manual_seed(31)
    net = torch.nn.ModuleDict(dict(backbone=Backbone(C), epi=epi.Epipolar(cfg=cfg), head=torch.nn.Conv2d(C, J, 1))).cuda().train()
    net["epi"].load_state_dict({k: torch.from_numpy(v) for k, v in syn.z_bn_params(C, 7).items()}, strict=False)
    two = copy.deepcopy(net)
    KRT = syn.ring_cameras(V * N, 4 * H, seed=3, jitter=20.0).reshape(V, N, 3, 4)
    P = torch.from_numpy(KRT.astype(np.float32)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(32)
    img = torch.randn((V * N, 3, 4 * H, 4 * W), device="cuda", generator=gen)
    target = torch.randn((V * N, J, H, W), device="cuda", generator=gen)
    src = [[(v + 1) % V] for v in range(V)]
    q, u = pair_items(src, N)

    # the reference's step (modeling/model.py:240-247): backbone on other_img, then on img, then the fusion and the head
    other_feat = two["backbone"](img[u])
    feat = two["backbone"](img)
    ret, _, _, _ = two["epi"](feat, other_feat, P.flatten(0, 1), P.flatten(0, 1)[u])
    loss_two = F.mse_loss(two["head"](ret + feat), target)
    loss_two.backward()

    # one backbone pass over the views
    feats = net["backbone"](img).unflatten(0, (V, N))
    ret, _, _, _ = net["epi"].forward_views_train(feats, P, sources=src)
    loss_one = F.mse_loss(net["head"](ret[:, 0].flatten(0, 1) + feats.flatten(0, 1)), target)
    loss_one.backward()

    assert abs(loss_one.item() - loss_two.item()) <= 1e-4 * abs(loss_two.item())
    grads_two = dict(two.named_parameters())
    for name, p in net.named_parameters():
        assert p.grad is not None and grads_two[name].grad is not None, name
        if name == "epi.z.bias":
            # z feeds a training-mode BatchNorm, which removes any per-channel constant: this gradient is zero up to rounding in
            # both flows, so it is held to the scale of the z weight's gradient instead of its own
            scale = grads_two["epi.z.weight"].grad.abs().max().item()
            assert (p.grad - grads_two[name].grad).abs().max().item() <= 1e-4 * scale, name
            continue
        assert rel_max(p.grad.cpu().numpy(), grads_two[name].grad.cpu().numpy()) < 1e-4, name


# ---- 7. buffers -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gradients_written_over_poisoned_workspace(dtype, det):
    """dL/dfeats between guards of its dtype's sentinel, the workspace prefilled with 0x00 and then 0xFF bytes: every element
    is written, no guard is, the inputs come back unchanged and both runs give the same bits (on the default path the float
    atomics may reorder, so there the two runs agree to rounding)"""
    V, N, C, H, W, K = 3, 2, 17 if dtype == torch.float32 else 64, 11, 13, 40
    feats, P, kw = inputs(V, N, C, H, W, K, seed=40)
    feats = feats.to(dtype)
    attn, locs, src, sources = run_forward(feats, P, "duplicates", K, **kw)
    w_out, _ = loss_weights(attn, C, 41, with_attn=False)
    f4 = feats.flatten(0, 1)
    NP = attn.shape[0] * attn.shape[1] * N
    a4, g4, l4 = attn.reshape(NP, K, H, W), w_out.reshape(NP, C, H, W), locs.reshape(K, NP, H, W, 2)
    keep = [t.clone() for t in (f4, a4, g4, l4)]
    t = np.ascontiguousarray(src, dtype=np.int32)
    lib = _lib.load()
    results = []
    for fill in (0x00, 0xFF):
        gr = Guarded((V * N, C, H, W), dtype)
        b = bwd_params(f4, f4, a4, g4, K=K, locs_in=l4, grad_ref=gr.t, deterministic=det)
        b.feat_src = b.P_src = None
        b.N = N
        targs = (V, t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), t.shape[1])
        nbytes = lib.epi_fusion_views_backward_workspace_bytes(ctypes.byref(b), *targs)
        ws = poisoned(nbytes, fill)
        b.workspace, b.workspace_bytes = ws.data_ptr(), nbytes
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(lib.epi_fusion_views_backward_f32(ctypes.byref(b), *targs, stream), "epi_fusion_views_backward_f32")
        torch.cuda.synchronize()
        assert (ws[nbytes:] == fill).all(), "the guard behind the workspace was written"
        gr.check("grad_ref")
        results.append(gr.t.clone())
    for x, k in zip((f4, a4, g4, l4), keep):
        assert torch.equal(int_bits(x), int_bits(k)), "an input of the backward was modified"
    if det:
        assert torch.equal(int_bits(results[0]), int_bits(results[1]))
    e = fp64_grads(feats, locs, w_out, None, src).cpu().numpy()
    for r in results:
        assert rel_max(r.float().cpu().numpy(), e.reshape(r.shape)) < lowp_tol(dtype)
