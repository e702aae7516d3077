"""GPU: every view of a frame against every other view in one call (the views form, EpiFusionParams.n_views).  Reference view v
with its j-th other view u = j + (j >= v) must give, bit for bit, what `epipolar_fusion(feats[v], feats[u], P[v], P[u])` gives —
for every kernel variant, dtype, epilogue, layout and map size — and the frame-level multi-view test must equal the
reference's loop (modeling/model.py:213-239) run once per reference view.  Every case has N >= 1 items per view with cameras
of their own, so that the pair index p = (v·(V−1) + j)·N + n, the view items v·N + n and u·N + n name different items."""
import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from oracle import mpjpe_proxy
from tests.test_gpu_buffers import Guarded, int_bits, poisoned
from tests.util import fusion_params, launch, workspace_bytes

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT_IDS = ["fp32", "bf16", "fp16"]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def view_inputs(V, N, C, H, W, K, seed=0):
    """-> feats [V,N,C,H,W], P [V,N,3,4] (a ring of V·N cameras: view v of item n is camera v·N + n), kwargs"""
    KRT = syn.ring_cameras(V * N, int(max(H, W) * 4), seed=seed, jitter=20.0).reshape(V, N, 3, 4)
    f = syn.features(V * N, C, H, W, "randn", seed + 1).reshape(V, N, C, H, W)
    return dev(f), dev(KRT.astype(np.float32)), dict(K=K, correct_normalize=True)


def random_z(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, C, generator=g) / np.sqrt(C)).float().cuda(), (0.1 * torch.randn(C, generator=g)).float().cuda()


def others(V, v):
    return [j + (j >= v) for j in range(V - 1)]


def singles(feats, P, sample_locs_in=None, **kw):
    """the reference loop: one epipolar_fusion per (reference view, other view), stacked as [V,V−1,...]; locations [K,V,V−1,...]"""
    V = feats.shape[0]
    res = []
    for v in range(V):
        for j, u in enumerate(others(V, v)):
            locs = None if sample_locs_in is None else sample_locs_in[:, v, j].contiguous()
            res.append(epi.epipolar_fusion(feats[v], feats[u], P[v], P[u], sample_locs_in=locs, **kw))
    out = []
    for i, r in enumerate(zip(*res)):
        if r[0] is None:
            out.append(None)
            continue
        t = torch.stack(list(r)).unflatten(0, (V, V - 1))
        out.append(t.permute(2, 0, 1, *range(3, t.dim())) if i == 3 else t)
    return out


def assert_views_equal_singles(feats, P, state=None, **kw):
    kw.setdefault("want_locs", True)
    want = singles(feats, P, **kw)
    got = epi.epipolar_fusion_views(feats, P, state=state, **kw)
    torch.cuda.synchronize()
    for what, g, w in zip(("out", "corr_pos", "attn", "sample_locs"), got, want):
        if w is None:
            assert g is None, what
            continue
        assert g.shape == w.shape and g.dtype == torch.float32, what
        assert torch.equal(g, w), "%s differs: max |diff| %.3g" % (what, (g - w).abs().max().item())
    return got


def variant_supported(feats, P, variant, **kw):
    try:
        epi.epipolar_fusion(feats[0], feats[1], P[0], P[1], variant=variant, **kw)
        return True
    except RuntimeError as e:
        assert "does not support" in str(e)
        return False


# ---- bit-exactness against V·(V−1) single calls ----------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["auto", "pipe", "sector", "tile", "warp"])
@pytest.mark.parametrize("V", [2, 4, 5])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_variants_dtypes(dtype, V, variant):
    feats, P, kw = view_inputs(V, 2, 64, 32, 32, 32, seed=V)
    feats = feats.to(dtype)
    if not variant_supported(feats, P, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    assert_views_equal_singles(feats, P, variant=variant, **kw)


@pytest.mark.parametrize("epilogue", ["add_ref", "z+zres", "z+zres+add_ref"])
@pytest.mark.parametrize("variant", ["auto", "warp"])
@pytest.mark.parametrize("C", [64, 264])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_epilogues(dtype, C, variant, epilogue):
    """residuals read the pair's reference view feats[v][n]: the fused kernel's direct store, the transposition pass, the
    tensor-core z GEMM (C = 64) and the fp32 z epilogue (C = 264)"""
    feats, P, kw = view_inputs(3, 2, C, 16, 16, 16, seed=C)
    kw.update(add_ref_residual="add_ref" in epilogue, variant=variant)
    if epilogue.startswith("z"):
        kw.update(z_folded=random_z(C, C), z_residual=True)
    assert_views_equal_singles(feats.to(dtype), P, **kw)


@pytest.mark.parametrize("variant", ["auto", "tile", "warp"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_injected_sample_locs(dtype, variant):
    feats, P, kw = view_inputs(3, 2, 64, 24, 24, 16, seed=3)
    feats = feats.to(dtype)
    locs = epi.epipolar_fusion_views(feats, P, want_locs=True, **kw)[3]                # [K,V,V−1,N,H,W,2]
    g = torch.Generator(device="cuda").manual_seed(4)
    locs = (locs + 0.02 * (torch.rand(locs.shape, device="cuda", generator=g) - 0.5)).contiguous()   # off the fused geometry
    assert_views_equal_singles(feats, P, sample_locs_in=locs, variant=variant, want_locs=False, **kw)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", ["64x64_items64", "96x96_items32"])
def test_item_sizes(shape, dtype):
    """both work-item sizes of the pipelined kernel with the views pair count: 64-pixel items (the cfg2 shape, z + ZRESIDUAL +
    the caller residual) and 32-pixel items (96×96)"""
    if shape == "64x64_items64":
        feats, P, kw = view_inputs(4, 2, 256, 64, 64, 64, seed=9)
        kw.update(z_folded=random_z(256, 2), z_residual=True, add_ref_residual=True)
    else:
        feats, P, kw = view_inputs(4, 1, 64, 96, 96, 32, seed=10)
    for variant in ("pipe", "auto"):
        assert_views_equal_singles(feats.to(dtype), P, variant=variant, **kw)


def test_fusion_state_cache():
    """one FusionState: miss -> hit -> one view's cameras changed -> back; each call equals fresh single calls, and a changed
    view invalidates exactly the 2·(V−1) pairs it belongs to (their cache epochs move, no other pair's does)"""
    V, N = 4, 2
    feats, P, kw = view_inputs(V, N, 64, 32, 32, 32, seed=6)
    kw.update(z_folded=random_z(64, 3), z_residual=True, variant="pipe")
    Pb = P.clone()
    Pb[2] = P[2].flip(0)                                          # view 2 takes the cameras of other items
    st = epi.FusionState()
    NP = V * (V - 1) * N

    def epochs():
        return st.cache[:NP * 128].view(torch.int32).view(NP, 32)[:, 31].clone()

    involved = torch.zeros(V, V - 1, N, dtype=torch.bool)
    for v in range(V):
        for j, u in enumerate(others(V, v)):
            involved[v, j] = 2 in (v, u)
    involved = involved.flatten().cuda()
    assert int(involved.sum()) == 2 * (V - 1) * N
    prev = None
    for i, Pi in enumerate((P, P, Pb, Pb, P)):
        assert_views_equal_singles(feats, Pi, state=st, **kw)
        e = epochs()
        if prev is not None:
            moved = e != prev
            if i in (1, 3):
                assert not moved.any(), "step %d: an unchanged camera pair was rebuilt" % i
            else:
                assert torch.equal(moved, involved), "step %d: pairs rebuilt %s" % (i, moved.nonzero().flatten().tolist())
        prev = e


@pytest.mark.parametrize("layout", ["channels_last", "strided", "odd_13x19", "list_of_maps"])
def test_layouts(layout):
    """channels_last and strided views as feats (no copy), odd-sized maps, and a sequence of V maps"""
    V, N, C, H, W = 3, 2, 64, 32, 32
    if layout == "odd_13x19":
        H, W = 13, 19
    feats, P, kw = view_inputs(V, N, C, H, W, 16, seed=11)
    if layout == "channels_last":
        feats = feats.flatten(0, 1).contiguous(memory_format=torch.channels_last).unflatten(0, (V, N))
    elif layout == "strided":
        big = torch.zeros(V, N, 2 * C, H, W + 3, device="cuda")
        big[:, :, ::2, :, :W] = feats
        feats = big[:, :, ::2, :, :W]
    for variant in ("auto", "warp"):
        want = singles(feats, P, variant=variant, want_locs=True, add_ref_residual=True, **kw)
        got = epi.epipolar_fusion_views(list(feats) if layout == "list_of_maps" else feats, P, variant=variant, want_locs=True,
                                        add_ref_residual=True, **kw)
        for what, g, w in zip(("out", "corr_pos", "attn", "sample_locs"), got, want):
            assert torch.equal(g, w), "%s %s" % (variant, what)


@pytest.mark.parametrize("case", ["pipe_z", "pipe_unstage_bf16", "warp_f16", "sector"])
def test_outputs_written_and_workspace_independent(case):
    """outputs between NaN-pattern guards, the workspace prefilled with 0x00 and then 0xFF: every output element is written,
    no guard is, and both runs give the same bits as the single calls"""
    variant, dtype, z = {"pipe_z": ("pipe", torch.float32, True), "pipe_unstage_bf16": ("pipe", torch.bfloat16, False),
                         "warp_f16": ("warp", torch.float16, False), "sector": ("sector", torch.float32, False)}[case]
    V, N, C, H, W, K = 3, 2, 64, 32, 32, 32
    feats, P, kw = view_inputs(V, N, C, H, W, K, seed=12)
    feats = feats.to(dtype)
    zw = random_z(C, 5) if z else None
    NP = V * (V - 1) * N
    f = feats.flatten(0, 1)
    runs = []
    for fill in (0x00, 0xFF):
        outs = dict(out=Guarded((NP, C, H, W)), attn=Guarded((NP, K, H, W)), corr=Guarded((NP, H, W, 2)),
                    locs=Guarded((K, NP, H, W, 2)))
        p = fusion_params(f, f, outs["out"].t, K=K, P1=P.reshape(V * N, 3, 4), attn=outs["attn"].t, corr=outs["corr"].t,
                          locs_out=outs["locs"].t, z=zw, z_residual=z, add_ref=True, variant=variant)
        p.N, p.n_views, p.feat_src, p.P_src = N, V, None, None
        nbytes = workspace_bytes(p)
        ws = poisoned(nbytes, fill)
        launch(p, ws)
        assert (ws[nbytes:] == fill).all(), "the guard behind the workspace was written"
        for k, g in outs.items():
            g.check("%s (workspace 0x%02X)" % (k, fill))
        runs.append({k: g.t.clone() for k, g in outs.items()})
    for k in runs[0]:
        assert torch.equal(int_bits(runs[0][k]), int_bits(runs[1][k])), "%s depends on the workspace's old contents" % k
    want = singles(feats, P, variant=variant, want_locs=True, add_ref_residual=True, z_folded=zw, z_residual=z, **kw)
    for k, w in zip(("out", "corr", "attn", "locs"), want):
        g = runs[0][k]
        assert torch.equal(g, w.flatten(1, 3) if k == "locs" else w.flatten(0, 2)), k


def test_inference_only():
    feats, P, kw = view_inputs(2, 1, 16, 12, 12, 8, seed=8)
    with pytest.raises(RuntimeError, match="epipolar_fusion"):
        epi.epipolar_fusion_views(feats.requires_grad_(True), P, **kw)
    with torch.no_grad():
        epi.epipolar_fusion_views(feats, P, **kw)


# ---- the module and the frame-level multi-view test ------------------------------------------------------------------------
@pytest.mark.parametrize("fuse_ref", [False, True])
def test_forward_views_equals_forward_loop(fuse_ref):
    cfg = epi.cfg_h36m_r50_256()
    cfg.VIS.EPIPOLAR_LINE = True
    m = epi.Epipolar(cfg=cfg, fuse_ref_residual=fuse_ref).cuda().eval()
    params = syn.z_bn_params(cfg.KEYPOINT.NFEATS, 5)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    C, (H, W) = cfg.KEYPOINT.NFEATS, cfg.KEYPOINT.HEATMAP_SIZE
    V = 4
    feats, P, _ = view_inputs(V, 1, C, H, W, cfg.EPIPOLAR.SAMPLESIZE, seed=12)
    with torch.no_grad():
        want = [[m(feats[v], feats[u], P[v], P[u]) for u in others(V, v)] for v in range(V)]
        for _ in range(2):                                      # alternate with forward: each keeps its own cached state
            got = m.forward_views(feats, P)
            again = m(feats[0], feats[1], P[0], P[1])
    assert len(m._states) == 2
    for i, what in enumerate(("finalout", "corr_pos", "attn", "sample_locs")):
        w = torch.stack([torch.stack([x[i] for x in row]) for row in want])
        assert torch.equal(got[i], w), what
        assert torch.equal(again[i], want[0][0][i]), what
    m.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        m.forward_views(feats, P)


@pytest.mark.parametrize("fuse_ref", [False, True])
def test_multitest_views_equals_reference_loop(fuse_ref):
    """every view of the proxy scene is the reference in turn; the result equals modeling/model.py:213-239 restated with
    single-source calls, run once per reference view, with the winning source reported as its camera index"""
    d = mpjpe_proxy.build(seed=0)
    V = mpjpe_proxy.V
    sampler = epi.Epipolar(cfg=d["cfg"], fuse_ref_residual=fuse_ref).cuda().eval()
    conv = torch.nn.Conv2d(mpjpe_proxy.C, mpjpe_proxy.J, 1, bias=False).cuda()
    conv.weight.data.copy_(torch.from_numpy(d["head"])[:, :, None, None])

    def tail(x):                                                # per item, so batch size cannot change the head's arithmetic
        return torch.cat([conv(x[i:i + 1]) for i in range(x.shape[0])])

    feat = dev(d["feat_ref"])                                   # [V,C,H,W]: view v of one frame
    KRT = dev(d["KRT"].astype(np.float32))
    feats, P = feat[:, None], KRT[:, None]                      # [V,1,...]: N = 1 item per view
    sigma, ds = 2.0, 4.0
    locs, scores, src = epi.multitest_views(sampler, tail, feats, P, sigma, ds)
    assert locs.shape[:2] == scores.shape[:2] == src.shape[:2] == (V, 1)
    with torch.no_grad():
        for v in range(V):
            all_locs, all_scos = [], []
            for u in others(V, v):
                ret, _, _, _ = epi.fused_other_feat(feats[v], feats[u], P[v], P[u], sampler)
                bl, bs = epi.find_tensor_peak_batch(tail(ret), sigma, ds)
                all_locs.append(bl); all_scos.append(bs)
            all_locs, all_scos = torch.stack(all_locs), torch.stack(all_scos)
            best, idx = torch.max(all_scos, 0)
            want = torch.gather(all_locs, 0, idx[None, ..., None].expand((-1, -1, -1, 2)))[0]
            cam = torch.tensor(others(V, v), device=idx.device)[idx]
            assert torch.equal(locs[v], want) and torch.equal(scores[v], best) and torch.equal(src[v], cam), v
    assert len(set(src.flatten().tolist())) > 1
