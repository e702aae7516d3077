"""GPU: the heat-map forward (epi_fusion_heatmaps_f32, `head=` on the functional forms and the module, `fuse_head=True` on the
test helpers).  The pose head's 1x1 conv runs as the fused forward's epilogue:
  heat = A·X + B·R + b,  A = Wh·(Wf + z_res·I),  B = Wh (0 without the caller's residual),  b = Wh·bf + bh.
Each heat element is an fp32 sum of 2C + 1 terms in one fixed order, so against the fp64 chain built on the library's own fused
feature X (a plain call without z and residual) it is held to the standard bound of such a sum plus the one rounding of A:
  |heat − heat64| <= (2C + 2)·2^-24·(|A|·|X| + |B|·|R| + |b|)   elementwise,
which scales with the magnitudes and so holds under cancellation in random heads."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, multiview
from oracle import c_oracle
from tests.test_gpu_buffers import Guarded, poisoned
from tests.test_gpu_views import DT_IDS, DTYPES, dev, random_z, view_inputs
from tests.test_gpu_view_sources import _proxy

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
VARIANTS = ["auto", "pipe", "sector", "tile", "warp"]


def head(J, C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(J, C, generator=g) / C ** 0.5).cuda(), torch.randn(J, generator=g).cuda()


def form_args(form, V, N):
    """(call kind, sources): pair, n_src = 3, views (all others), [V,1] and [V,2] tables"""
    return {"pair": ("pair", None), "nsrc3": ("multi", None), "views": ("views", None),
            "table1": ("views", [[(v + 1) % V] for v in range(V)]),
            "table2": ("views", [[(v + 1) % V, (v + V - 1) % V] for v in range(V)])}[form]


def run(form, feats, P, **kw):
    """the call of `form` on view maps feats [V,N,C,H,W] -> (first result flattened to pairs, corr, attn, locs, residual items
    [pairs,C,H,W]: the pair's query item)"""
    V, N = feats.shape[:2]
    kind, src = form_args(form, V, N)
    if kind == "pair":
        r = epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], **kw)
        return r[0], r[1], r[2], r[3], feats[0]
    if kind == "multi":
        r = epi.epipolar_fusion_multi(feats[0], feats[1:4], P[0], P[1:4], **kw)
        return r[0].flatten(0, 1), r[1], r[2], r[3], feats[0].repeat(3, 1, 1, 1)
    r = epi.epipolar_fusion_views(feats, P, sources=src, **kw)
    S = r[0].shape[1]
    return r[0].flatten(0, 2), r[1], r[2], r[3], feats[:, None].expand(V, S, *feats.shape[1:]).flatten(0, 2)


def heat64(X, R, Wh, bh, z, zres, residual):
    """fp64 chain on the library's fused feature X [P,C,H,W] and the residual items R -> (heat64, bound)"""
    d = lambda t: t.double().cpu()
    X, R, Wh, bh = d(X), d(R), d(Wh), d(bh)
    C = X.shape[1]
    if z is not None:
        Wf, bf = d(z[0]), d(z[1])
        A = Wh @ (Wf + (torch.eye(C, dtype=torch.float64) if zres else 0))
        b = Wh @ bf + bh
    else:
        A, b = Wh, bh
    B = Wh if residual else torch.zeros_like(Wh)
    mm = lambda M, T: torch.einsum("jc,pchw->pjhw", M, T)
    h = mm(A, X) + mm(B, R) + b[None, :, None, None]
    bound = (2 * C + 2) * U * (mm(A.abs(), X.abs()) + mm(B.abs(), R.abs()) + b.abs()[None, :, None, None])
    return h, bound


def conv64(conv, x):
    """the 1x1 conv in fp64 (PyTorch's own may run in TF32)"""
    w = conv.weight.detach().double().cpu().flatten(1)
    b = 0 if conv.bias is None else conv.bias.detach().double().cpu()[None, :, None, None]
    return torch.einsum("jc,nchw->njhw", w, x.double().cpu()) + b


def check_fp64(form, variant, dtype=torch.float32, z_mode="zres", residual=True, J=17, C=64, H=16, W=16, K=16, N=2, seed=0,
               out_dtype=torch.float32):
    V = 4
    feats, P, kw = view_inputs(V, N, C, H, W, K, seed=seed)
    feats = feats.to(dtype)
    Wh, bh = head(J, C, seed + 7)
    z = None if z_mode == "noz" else random_z(C, seed + 3)
    zres = z_mode == "zres"
    try:
        X, corr0, attn0, locs0, R = run(form, feats, P, variant=variant, want_locs=True, **kw)
    except RuntimeError as e:
        assert "does not support" in str(e)
        pytest.skip("%s does not run this shape" % variant)
    heat, corr, attn, locs, _ = run(form, feats, P, variant=variant, want_locs=True, z_folded=z, z_residual=zres,
                                    add_ref_residual=residual, head=(Wh, bh), out_dtype=out_dtype, **kw)
    torch.cuda.synchronize()
    for g, w in ((corr, corr0), (attn, attn0), (locs, locs0)):       # the plain call's outputs, bit for bit
        assert torch.equal(g, w)
    assert heat.dtype == out_dtype and heat.shape == (X.shape[0], J, H, W)
    h64, bound = heat64(X, R, Wh, bh, z, zres, residual)
    err = (heat.double().cpu() - h64).abs()
    if out_dtype == torch.float32:
        assert (err <= bound).all(), "max err/bound %.3g" % (err / bound.clamp_min(1e-300)).max().item()
    return heat


# ---- against fp64 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("form", ["pair", "nsrc3", "views", "table1", "table2"])
def test_fp64_forms_variants(form, variant):
    check_fp64(form, variant)


@pytest.mark.parametrize("residual", [True, False], ids=["res", "nores"])
@pytest.mark.parametrize("z_mode", ["zres", "z", "noz"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_fp64_epilogue_options(dtype, z_mode, residual):
    check_fp64("table1", "auto", dtype=dtype, z_mode=z_mode, residual=residual)


@pytest.mark.parametrize("J", [1, 17, 20, 64])
@pytest.mark.parametrize("C", [12, 64, 256, 264])
def test_fp64_joints_channels(J, C):
    check_fp64("pair", "auto", J=J, C=C, N=1)


@pytest.mark.parametrize("variant", VARIANTS)
def test_fp64_odd_map(variant):
    check_fp64("views", variant, H=13, W=21)


# ---- contracts: bit equality across forms, 16-bit heat = fp32 heat rounded once -----------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_forms_bit_equal_pair_form(dtype):
    V, N, C, J = 4, 2, 64, 20
    feats, P, kw = view_inputs(V, N, C, 16, 16, 16, seed=4)
    feats = feats.to(dtype)
    Wh, bh = head(J, C, 5)
    z = random_z(C, 6)
    kw.update(z_folded=z, z_residual=True, add_ref_residual=True, head=(Wh, bh))
    pair = lambda v, u: epi.epipolar_fusion(feats[v], feats[u], P[v], P[u], **kw)[0]
    src = [[(v + 1) % V, (v + 2) % V] for v in range(V)]
    heat = epi.epipolar_fusion_views(feats, P, sources=src, **kw)[0]
    allh = epi.epipolar_fusion_views(feats, P, **kw)[0]
    multi = epi.epipolar_fusion_multi(feats[0], feats[1:], P[0], P[1:], **kw)[0]
    for v in range(V):
        for j, u in enumerate(src[v]):
            assert torch.equal(heat[v, j], pair(v, u))
        for j in range(V - 1):
            assert torch.equal(allh[v, j], pair(v, j + (j >= v)))
    for s in range(V - 1):
        assert torch.equal(multi[s], pair(0, s + 1))


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("variant", ["pipe", "warp"])
def test_16bit_heat_is_fp32_rounded_once(out_dtype, variant):
    h32 = check_fp64("table2", variant, dtype=torch.bfloat16)
    h16 = check_fp64("table2", variant, dtype=torch.bfloat16, out_dtype=out_dtype)
    assert torch.equal(h16, h32.to(out_dtype))


# ---- end to end: the C oracle and fp64 attention ------------------------------------------------------------------------------
def test_module_against_oracle():
    N, C, H, W, K, J = 2, 64, 32, 32, 32, 17
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True),
                       VIS=dict(EPIPOLAR_LINE=True))
    feats, P, _ = view_inputs(2, N, C, H, W, K, seed=9)
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    conv = torch.nn.Conv2d(C, J, 1).cuda()
    with torch.no_grad():
        heat, corr, attn, locs = m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)
        ret, corr0, attn0, locs0 = m(feats[0], feats[1], P[0], P[1])
        want = conv64(conv, ret + feats[0])
    assert torch.equal(corr, corr0) and torch.equal(attn, attn0) and torch.equal(locs, locs0)
    o = c_oracle.forward(cfg, feats[0].cpu().numpy(), feats[1].cpu().numpy(), P[0].cpu().numpy(), P[1].cpu().numpy(),
                         locs=locs.transpose(0, 1).contiguous().cpu().numpy())
    ref = conv64(conv, torch.from_numpy(o["out"]).double() + feats[0].double().cpu())
    assert ((heat.double().cpu() - ref).abs().max() / ref.abs().max()).item() < 1e-4
    assert np.abs(attn.cpu().numpy() - o["attn"]).max() < 1e-5
    assert ((heat.double().cpu() - want).abs().max() / want.abs().max()).item() < 1e-5    # the head on the unfused feature


# ---- layouts: channels-last residual, strided heat through the C ABI ----------------------------------------------------------
def heat_call(f1, f2, P1, P2, A, B, b, heat, K=16, variant="auto", workspace=None, cache=None, fill=None):
    from tests.util import fusion_params
    lib = _lib.load()
    p = fusion_params(f1, f2, f1, K=K, P1=P1, P2=P2, variant=variant)
    p.out = None
    p.feat_dtype = p.feat_dtype | _lib.EPI_OUT_DTYPE({torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[heat.dtype])
    h = _lib.EpiHeadParams()
    h.A, h.B, h.b = A.data_ptr(), None if B is None else B.data_ptr(), b.data_ptr()
    h.heat, h.heat_stride, h.J = heat.data_ptr(), (ctypes.c_int64 * 4)(*heat.stride()), A.shape[0]
    nbytes = lib.epi_fusion_heatmaps_workspace_bytes(ctypes.byref(p), ctypes.byref(h), None, 0)
    if workspace is None:
        workspace = torch.empty(max(nbytes, 1), device="cuda", dtype=torch.uint8)
    p.workspace, p.workspace_bytes = workspace.data_ptr(), nbytes
    if cache is not None:
        p.cache, p.cache_bytes = cache.data_ptr(), cache.numel()
    _lib.check(lib.epi_fusion_heatmaps_f32(ctypes.byref(p), ctypes.byref(h), None, 0,
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "epi_fusion_heatmaps_f32")
    torch.cuda.synchronize()
    return lib.epi_last_launch_count(), nbytes


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("variant", ["pipe", "warp"])
def test_channels_last_residual_strided_heat_poisoned_workspace(dtype, variant):
    N, C, H, W, J = 2, 64, 13, 21, 20
    feats, P, kw = view_inputs(2, N, C, H, W, 16, seed=11)
    feats = feats.to(dtype)
    Wh, bh = head(J, C, 12)
    A, b = epi.fold_head(Wh, bh)
    want = epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], variant=variant, add_ref_residual=True, head=(Wh, bh), **kw)[0]
    f1 = feats[0].contiguous(memory_format=torch.channels_last)
    heat_buf = Guarded((N, J, H, W + 3), torch.float32)               # a strided view of a wider buffer
    heat = heat_buf.t[..., 1:W + 1]
    for fill in (0x00, 0xff):
        heat_buf.t.fill_(float("nan"))
        ws = poisoned(64 << 20, fill)
        n, nbytes = heat_call(f1, feats[1], P[0], P[1], A, Wh.contiguous(), b, heat, variant=variant, workspace=ws)
        assert nbytes < (64 << 20)
        assert torch.equal(heat, want), fill
        assert (ws[nbytes:] == fill).all(), "a workspace byte past its size was written"
        assert heat_buf.t[..., 0].isnan().all() and heat_buf.t[..., W + 1:].isnan().all()


# ---- launches and the FusionState cache --------------------------------------------------------------------------------------
def test_launch_count_and_cache():
    N, C, H, W, K, J = 4, 256, 64, 64, 64, 17                           # cfg2's shape: staging, fused kernel, head
    feats, P, _ = view_inputs(2, N, C, H, W, K, seed=13)
    Wh, bh = head(J, C, 14)
    A, b = epi.fold_head(Wh, bh)
    heat = torch.empty(N, J, H, W, device="cuda")
    n, _ = heat_call(feats[0], feats[1], P[0], P[1], A, Wh, b, heat, K=K)
    assert n == 3
    st = epi.FusionState()
    kw = dict(K=K, correct_normalize=True, add_ref_residual=True, head=(Wh, bh))
    fresh = lambda P1, P2: epi.epipolar_fusion(feats[0], feats[1], P1, P2, **kw)[0]
    miss = epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], state=st, **kw)[0]
    hit = epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], state=st, **kw)[0]
    assert st.cache is not None
    assert torch.equal(miss, fresh(P[0], P[1])) and torch.equal(hit, miss)
    moved = epi.epipolar_fusion(feats[0], feats[1], P[1], P[0], state=st, **kw)[0]     # a camera change on the same cache
    assert torch.equal(moved, fresh(P[1], P[0])) and not torch.equal(moved, miss)


def test_module_heat_cached_fold_graph_and_half():
    N, C, H, W, K, J = 2, 64, 16, 16, 16, 17
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True,
                                                                                   PARAMETERIZED=["z"], ZRESIDUAL=True))
    feats, P, _ = view_inputs(2, N, C, H, W, K, seed=15)
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    with torch.no_grad():
        m.bn.weight.normal_(); m.bn.bias.normal_(); m.bn.running_mean.normal_(); m.bn.running_var.uniform_(0.5, 2)
    conv = torch.nn.Conv2d(C, J, 1).cuda()
    with torch.no_grad():
        h1 = m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)[0]
        ref = conv64(conv, m(feats[0], feats[1], P[0], P[1])[0] + feats[0])
        assert ((h1.double().cpu() - ref).abs().max() / ref.abs().max()).item() < 1e-5
        h2 = m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)[0]
        assert torch.equal(h1, h2)
        conv.weight.mul_(2)                                            # a new parameter version refolds
        assert not torch.equal(m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)[0], h1)
        conv.weight.div_(2)
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)
            with torch.cuda.graph(g, stream=s):
                hg = m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)[0]
        torch.cuda.current_stream().wait_stream(s)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(hg, h1)
        mh = m.to(torch.bfloat16)
        hb = mh.forward_heatmaps(feats[0].bfloat16(), feats[1].bfloat16(), P[0], P[1], conv)[0]
        assert hb.dtype == torch.bfloat16
        m.train()
        with pytest.raises(RuntimeError, match="eval"):
            m.forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)
    with pytest.raises(RuntimeError, match="inference only"):
        m.eval().float().forward_heatmaps(feats[0], feats[1], P[0], P[1], conv)      # conv.weight requires grad


# ---- the MPJPE proxy scene: the three helpers, fused head against the unfused tail ---------------------------------------------
def same_peaks(a, b):
    """locs within 1e-3 px and the same source view, except where the sources' best scores tie (1e-5 relative): the ring's two
    neighbours of a view see it alike, and another fp32 sum order could pick the other one (none does on this scene)"""
    same = a[2] == b[2]
    assert ((a[0] - b[0]).abs().amax(-1)[same] <= 1e-3).all()
    tie = (a[1] - b[1]).abs() <= 1e-5 * a[1].abs()
    assert (same | tie).all(), "a different source without a tie of the scores"
    return int((~same).sum())


def test_mpjpe_proxy_helpers_fused_head():
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):     # the unfused tail in fp32, as the fused head
        mpjpe_proxy_helpers()


def mpjpe_proxy_helpers():
    sampler, tail, feats, P, KRT = _proxy(False)
    conv = next(c.cell_contents for c in tail.__closure__ if isinstance(c.cell_contents, torch.nn.Conv2d))
    V = feats.shape[0]
    sigma, ds = 2.0, 4.0
    src = multiview.nearest_view_table(KRT, topk=1)
    a = epi.standard_views_test(sampler, conv, feats, P, src, sigma, ds)
    b = epi.standard_views_test(sampler, conv, feats, P, src, sigma, ds, fuse_head=True)
    assert (a[0] - b[0]).abs().max().item() <= 1e-3
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
    src2 = multiview.nearest_view_table(KRT, topk=2)
    flips = 0
    for sources in (None, src2):
        a = epi.multitest_views(sampler, conv, feats, P, sigma, ds, sources=sources)
        b = epi.multitest_views(sampler, conv, feats, P, sigma, ds, sources=sources, fuse_head=True)
        flips += same_peaks(a, b)
    others = torch.stack([feats[u] for u in range(1, V)])
    Po = torch.stack([P[u] for u in range(1, V)])
    a = epi.multitest(sampler, conv, feats[0], others, P[0], Po, sigma, ds)
    b = epi.multitest(sampler, conv, feats[0], others, P[0], Po, sigma, ds, fuse_head=True)
    flips += same_peaks(a, b)
    print("joints whose tied sources flipped: %d" % flips)
