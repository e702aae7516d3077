"""GPU: several source views per reference item in one call (the reference's MULTITEST path, modeling/model.py:213-239).
Source s of reference item n must give, bit for bit, what a single-source call on (feat_ref, feat_srcs[s]) gives — for every
kernel variant, layout, dtype and epilogue — and the best-source peak selection must equal torch.max + gather over the
single-source peak finder.  Every case has N >= 2 and S = 3 with a distinct map and distinct cameras per source, so that the
pair index p = s·N + n, p % N and p / S name different items."""
import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from oracle import mpjpe_proxy

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT_IDS = ["fp32", "bf16", "fp16"]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def multi_inputs(N, C, H, W, K, S=3, cams="ring", seed=0):
    """-> feat_ref [N,C,H,W], feat_srcs [S,N,C,H,W], P_ref [N,3,4], P_srcs [S,N,3,4], kwargs.  Ring cameras: reference item n
    is view n of N + S views and its source s is view (n + 1 + s) mod (N + S); 'randn': literal random KRTs (lines that miss
    the image)."""
    if cams == "ring":
        V = N + S
        KRT = syn.ring_cameras(V, int(max(H, W) * 4), seed=seed, jitter=20.0)
        P1 = KRT[:N]
        P2 = np.stack([KRT[[(n + 1 + s) % V for n in range(N)]] for s in range(S)])
    else:
        rng = np.random.default_rng(seed + 31)
        P1, P2 = rng.standard_normal((N, 3, 4)), rng.standard_normal((S, N, 3, 4))
    f1 = syn.features(N, C, H, W, "randn", seed + 1)
    f2 = syn.features(S * N, C, H, W, "randn", seed + 2).reshape(S, N, C, H, W)
    return dev(f1), dev(f2), dev(P1.astype(np.float32)), dev(P2.astype(np.float32)), dict(K=K, correct_normalize=cams == "ring")


def random_z(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, C, generator=g) / np.sqrt(C)).float().cuda(), (0.1 * torch.randn(C, generator=g)).float().cuda()


def to_layout(t, channels_last):
    if not channels_last:
        return t
    if t.dim() == 4:
        return t.contiguous(memory_format=torch.channels_last)
    return t.flatten(0, 1).contiguous(memory_format=torch.channels_last).unflatten(0, tuple(t.shape[:2]))


def singles(f1, f2, P1, P2, sample_locs_in=None, out_cl=False, **kw):
    """the reference loop: one epipolar_fusion per source, stacked"""
    res = []
    for s in range(f2.shape[0]):
        o = None if not out_cl else torch.empty_like(f1, dtype=torch.float32, memory_format=torch.channels_last)
        locs_s = None if sample_locs_in is None else sample_locs_in[:, s].contiguous()
        res.append(epi.epipolar_fusion(f1, f2[s], P1, P2[s], sample_locs_in=locs_s, out=o, **kw))
    return [None if r[0] is None else torch.stack(list(r)) for r in zip(*res)]


def assert_multi_equals_singles(f1, f2, P1, P2, out_cl=False, state=None, **kw):
    kw.setdefault("want_locs", True)
    want = singles(f1, f2, P1, P2, out_cl=out_cl, **kw)
    S, N, C, H, W = f2.shape
    out = None
    if out_cl:
        out = torch.empty(S * N, C, H, W, device=f1.device).contiguous(memory_format=torch.channels_last).unflatten(0, (S, N))
    got = epi.epipolar_fusion_multi(f1, f2, P1, P2, out=out, state=state, **kw)
    torch.cuda.synchronize()
    # the multi-source locations are [K,S,N,H,W,2]; the stacked single-source ones [S,K,N,H,W,2]
    want[3] = None if want[3] is None else want[3].transpose(0, 1)
    for what, g, w in zip(("out", "corr_pos", "attn", "sample_locs"), got, want):
        if w is None:
            assert g is None, what
            continue
        assert g.shape == w.shape and g.dtype == torch.float32, what
        assert torch.equal(g, w), "%s differs: max |diff| %.3g" % (what, (g - w).abs().max().item())
    return got


def variant_supported(f1, f2, P1, P2, variant, **kw):
    try:
        epi.epipolar_fusion(f1, f2[0], P1, P2[0], variant=variant, **kw)
        return True
    except RuntimeError as e:
        assert "does not support" in str(e)
        return False


# ---- bit-exactness against S single-source calls -------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("variant", ["auto", "pipe", "sector", "tile", "warp"])
@pytest.mark.parametrize("cams", ["ring", "randn"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_variants_layouts_dtypes(dtype, cams, variant, layout):
    f1, f2, P1, P2, kw = multi_inputs(2, 64, 32, 32, 32, cams=cams, seed=5)
    cl = layout == "channels_last"
    f1, f2 = to_layout(f1.to(dtype), cl), to_layout(f2.to(dtype), cl)
    if not variant_supported(f1, f2, P1, P2, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    assert_multi_equals_singles(f1, f2, P1, P2, out_cl=cl, variant=variant, **kw)


@pytest.mark.parametrize("out_layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("epilogue", ["none", "add_ref", "z", "z+zres", "z+zres+add_ref"])
@pytest.mark.parametrize("variant", ["auto", "warp"])
@pytest.mark.parametrize("C", [64, 264])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_epilogues(dtype, C, variant, epilogue, out_layout):
    """Residuals read feat_ref[n] and ZRESIDUAL adds pair p's own feature in every epilogue: the fused kernel's direct store,
    the transposition pass, the tensor-core z GEMM (C = 64) and the fp32 z epilogue (C = 264)."""
    f1, f2, P1, P2, kw = multi_inputs(2, C, 16, 16, 16, seed=C)
    f1, f2 = f1.to(dtype), f2.to(dtype)
    kw.update(add_ref_residual="add_ref" in epilogue, variant=variant)
    if epilogue.startswith("z"):
        kw.update(z_folded=random_z(C, C), z_residual="zres" in epilogue)
    assert_multi_equals_singles(f1, f2, P1, P2, out_cl=out_layout == "channels_last", **kw)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_cfg2_z_zresidual(dtype):
    """the benchmark's workload: N=4, C=256, 64x64, K=64, z + ZRESIDUAL + the caller residual"""
    f1, f2, P1, P2, kw = multi_inputs(4, 256, 64, 64, 64, seed=9)
    assert_multi_equals_singles(f1.to(dtype), f2.to(dtype), P1, P2, z_folded=random_z(256, 2), z_residual=True,
                                add_ref_residual=True, **kw)


@pytest.mark.parametrize("variant", ["auto", "tile", "warp"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_injected_sample_locs(dtype, variant):
    f1, f2, P1, P2, kw = multi_inputs(2, 64, 24, 24, 16, seed=3)
    f1, f2 = f1.to(dtype), f2.to(dtype)
    locs = epi.epipolar_fusion_multi(f1, f2, P1, P2, want_locs=True, **kw)[3]          # [K,S,N,H,W,2]
    g = torch.Generator(device="cuda").manual_seed(4)
    locs = (locs + 0.02 * (torch.rand(locs.shape, device="cuda", generator=g) - 0.5)).contiguous()   # off the fused geometry
    want = singles(f1, f2, P1, P2, sample_locs_in=locs, variant=variant, **kw)
    got = epi.epipolar_fusion_multi(f1, f2, P1, P2, sample_locs_in=locs, variant=variant, **kw)
    for what, g_, w in zip(("out", "corr_pos", "attn"), got, want):
        assert torch.equal(g_, w), what


# (N, C, H, W, K), variant: a C % 8 != 0 shape only the warp kernel takes, and a map above 16384 pixels (row-windowed union
# bitmap of the pipelined kernel, pixel order in a launch of its own)
SHAPES = {"warp_c12": ((2, 12, 12, 20, 16), "warp"), "pipe_132x136": ((2, 64, 132, 136, 16), "pipe")}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_shape_envelope(dtype, shape):
    (N, C, H, W, K), variant = SHAPES[shape]
    f1, f2, P1, P2, kw = multi_inputs(N, C, H, W, K, seed=C)
    f1, f2 = f1.to(dtype), f2.to(dtype)
    for v in (variant, "auto"):
        assert_multi_equals_singles(f1, f2, P1, P2, variant=v, add_ref_residual=True, **kw)


def test_sequence_of_maps_and_single_source():
    """feat_srcs as a list of S maps; S = 1 equals epipolar_fusion"""
    f1, f2, P1, P2, kw = multi_inputs(2, 64, 32, 32, 32, seed=1)
    a = epi.epipolar_fusion_multi(f1, list(f2), P1, P2, **kw)
    b = epi.epipolar_fusion_multi(f1, f2, P1, P2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a[:3], b[:3]))
    one = epi.epipolar_fusion_multi(f1, f2[:1], P1, P2[:1], **kw)
    ref = epi.epipolar_fusion(f1, f2[0], P1, P2[0], **kw)
    assert all(torch.equal(x[0], y) for x, y in zip(one[:3], ref[:3]))


def test_n_src_zero_and_one_are_todays_call():
    """n_src = 1 in the parameter block gives the same bits as n_src = 0 (the default of every existing caller)"""
    f1, f2, P1, P2, kw = multi_inputs(2, 64, 32, 32, 32, seed=2)
    kw.update(z_folded=random_z(64, 1), z_residual=True, add_ref_residual=True, want_locs=True)
    want = epi.epipolar_fusion(f1, f2[0], P1, P2[0], **kw)
    st = epi.FusionState()
    got0 = [t.clone() for t in epi.epipolar_fusion(f1, f2[0], P1, P2[0], state=st, **kw)]
    assert st.params.n_src == 0
    st.params.n_src = 1                                         # same key: the next call re-uses this parameter block
    got1 = epi.epipolar_fusion(f1, f2[0], P1, P2[0], state=st, **kw)
    for w, g0, g1 in zip(want, got0, got1):
        assert torch.equal(g0, w) and torch.equal(g1, w)


def test_fusion_state_with_sources():
    """one FusionState: miss -> hit -> one source's cameras changed -> back; each call equals a fresh loop of single calls"""
    f1, f2, P1, P2, kw = multi_inputs(2, 64, 32, 32, 32, seed=6)
    kw.update(z_folded=random_z(64, 3), z_residual=True)
    P2b = P2.clone()
    P2b[1] = P2[2].flip(0)                                      # source 1 takes other cameras
    st = epi.FusionState()
    for P in (P2, P2, P2b, P2b, P2):
        assert_multi_equals_singles(f1, f2, P1, P, state=st, **kw)
    # the key includes S: a two-source call on the same state re-plans instead of reading three-source records
    assert_multi_equals_singles(f1, f2[:2], P1, P2[:2], state=st, **kw)


def test_inference_only():
    f1, f2, P1, P2, kw = multi_inputs(2, 16, 12, 12, 8, seed=8)
    with pytest.raises(RuntimeError, match="epipolar_fusion"):
        epi.epipolar_fusion_multi(f1.requires_grad_(True), f2, P1, P2, **kw)
    with torch.no_grad():
        epi.epipolar_fusion_multi(f1, f2, P1, P2, **kw)


# ---- the module ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fuse_ref", [False, True])
def test_forward_multi_equals_forward_loop(fuse_ref):
    cfg = epi.cfg_h36m_r50_256()
    cfg.VIS.EPIPOLAR_LINE = True
    m = epi.Epipolar(cfg=cfg, fuse_ref_residual=fuse_ref).cuda().eval()
    params = syn.z_bn_params(cfg.KEYPOINT.NFEATS, 5)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    C, (H, W) = cfg.KEYPOINT.NFEATS, cfg.KEYPOINT.HEATMAP_SIZE
    f1, f2, P1, P2, _ = multi_inputs(2, C, H, W, cfg.EPIPOLAR.SAMPLESIZE, seed=12)
    with torch.no_grad():
        want = [m(f1, f2[s], P1, P2[s]) for s in range(3)]
        for _ in range(2):                                      # alternate with forward: each keeps its own cached state
            got = m.forward_multi(f1, f2, P1, P2)
            again = m(f1, f2[0], P1, P2[0])
    assert len(m._states) == 2
    for i, what in enumerate(("finalout", "corr_pos", "attn", "sample_locs")):
        w = torch.stack([x[i] for x in want])
        assert torch.equal(got[i], w), what
        assert torch.equal(again[i], want[0][i]), what
    m.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        m.forward_multi(f1, f2, P1, P2)


# ---- best-source peaks --------------------------------------------------------------------------------------------------
def reference_best(heat, radius, ds):
    """modeling/model.py:229-234 over find_tensor_peak_batch"""
    locs, scos = zip(*[epi.find_tensor_peak_batch(h, radius, ds) for h in heat])
    all_locs, all_scos = torch.stack(locs), torch.stack(scos)
    best, idx = torch.max(all_scos, 0)
    return torch.gather(all_locs, 0, idx[None, ..., None].expand((-1, -1, -1, 2)))[0], best, idx


def test_peak_best_equals_max_gather():
    g = torch.Generator(device="cuda").manual_seed(0)
    heat = torch.rand(3, 4, 17, 64, 48, device="cuda", generator=g)
    locs, scores, src = epi.find_tensor_peak_best(heat, 2.0, 4.0)
    wl, ws, wi = reference_best(heat, 2.0, 4.0)
    assert torch.equal(locs, wl) and torch.equal(scores, ws) and torch.equal(src, wi)
    assert len(set(src.flatten().tolist())) == 3                # every source wins somewhere


def test_peak_best_tie_keeps_first_source():
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.rand(2, 5, 32, 32, device="cuda", generator=g)
    b = torch.rand(2, 5, 32, 32, device="cuda", generator=g) * 0.5
    heat = torch.stack([b, a, a])                               # sources 1 and 2 tie everywhere and beat source 0
    locs, scores, src = epi.find_tensor_peak_best(heat, 1.5, 4.0)
    wl, ws, wi = reference_best(heat, 1.5, 4.0)
    assert (src == 1).all() and torch.equal(src, wi)
    assert torch.equal(locs, wl) and torch.equal(scores, ws)


def test_peak_best_single_source_is_find_tensor_peak_batch():
    g = torch.Generator(device="cuda").manual_seed(2)
    heat = torch.randn(1, 3, 21, 40, 56, device="cuda", generator=g)
    locs, scores, src = epi.find_tensor_peak_best(heat, 3.0, 4.0)
    wl, ws = epi.find_tensor_peak_batch(heat[0], 3.0, 4.0)
    assert torch.equal(locs, wl) and torch.equal(scores, ws) and (src == 0).all()


# ---- the multi-view test on the MPJPE proxy scene -----------------------------------------------------------------------
@pytest.mark.parametrize("fuse_ref", [False, True])
def test_multitest_equals_reference_loop(fuse_ref):
    """every view of the proxy scene is a reference and the other three its sources; the fused multi-source path equals the
    reference's loop of modeling/model.py:213-239 restated with single-source calls"""
    d = mpjpe_proxy.build(seed=0)
    V = mpjpe_proxy.V
    sampler = epi.Epipolar(cfg=d["cfg"], fuse_ref_residual=fuse_ref).cuda().eval()
    conv = torch.nn.Conv2d(mpjpe_proxy.C, mpjpe_proxy.J, 1, bias=False).cuda()
    conv.weight.data.copy_(torch.from_numpy(d["head"])[:, :, None, None])

    def tail(x):                                                # per item, so batch size cannot change the head's arithmetic
        return torch.cat([conv(x[i:i + 1]) for i in range(x.shape[0])])

    feat = dev(d["feat_ref"])
    KRT = dev(d["KRT"].astype(np.float32))
    others = [[(v + 1 + s) % V for v in range(V)] for s in range(V - 1)]
    other_feats = torch.stack([feat[o] for o in others])
    other_KRTs = torch.stack([KRT[o] for o in others])
    sigma, ds = 2.0, 4.0
    locs, scores, src = epi.multitest(sampler, tail, feat, other_feats, KRT, other_KRTs, sigma, ds)
    with torch.no_grad():
        all_locs, all_scos = [], []
        for s in range(V - 1):
            ret, _, _, _ = epi.fused_other_feat(feat, other_feats[s], KRT, other_KRTs[s], sampler)
            bl, bs = epi.find_tensor_peak_batch(tail(ret), sigma, ds)
            all_locs.append(bl); all_scos.append(bs)
        all_locs, all_scos = torch.stack(all_locs), torch.stack(all_scos)
        best, idx = torch.max(all_scos, 0)
        want = torch.gather(all_locs, 0, idx[None, ..., None].expand((-1, -1, -1, 2)))[0]
    assert torch.equal(locs, want) and torch.equal(scores, best) and torch.equal(src, idx)
