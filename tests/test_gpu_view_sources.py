"""GPU: the views form with a caller's source table (`epipolar_fusion_views(..., sources=)`, the
epi_fusion_view_sources_* entry points).  View v with its j-th source u = sources[v][j] must give, bit for bit, what
`epipolar_fusion(feats[v], feats[u], P[v], P[u])` gives — for every kernel variant, dtype, epilogue, layout and table shape —
and the standard test (each view with its nearest camera) from one call must equal the reference's two-pass flow
(modeling/model.py:240-247, modeling/backbones/resnet.py:377-430).  Every case has N >= 1 items per view with cameras of their
own, so that the pair p = (v·S + j)·N + n, the query item v·N + n and the source item u·N + n are different items."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, multiview
from epipolar_transformers_b200 import synthetic as syn
from oracle import mpjpe_proxy
from tests.test_gpu_buffers import Guarded, int_bits, poisoned
from tests.test_gpu_views import DT_IDS, DTYPES, dev, others, random_z, variant_supported, view_inputs
from tests.util import fusion_params

pytestmark = pytest.mark.gpu
OUTS = ("out", "corr_pos", "attn", "sample_locs")


def table(kind, V):
    """[V,S] source tables: the nearest camera, two sources, a view nobody uses, a view everybody uses, duplicates"""
    if kind == "nearest":
        return [[(v + 1) % V] for v in range(V)]
    if kind == "s2":
        return [[(v + 1) % V, (v + V - 1) % V] for v in range(V)]
    if kind == "nobodys_source":                       # view 0 is nobody's source
        return [[2 if v == 1 else 1] for v in range(V)]
    if kind == "everybodys_source":                    # view 0 is every other view's only source
        return [[1 if v == 0 else 0] for v in range(V)]
    if kind == "duplicates":
        return [[(v + 1) % V, (v + 1) % V, (v + 2) % V if (v + 2) % V != v else (v + 1) % V] for v in range(V)]
    raise ValueError(kind)


TABLES = ["nearest", "s2", "nobodys_source", "everybodys_source", "duplicates"]


def singles(feats, P, sources, sample_locs_in=None, **kw):
    """the reference loop: one epipolar_fusion per (view, source), stacked as [V,S,...]; locations [K,V,S,...]"""
    V, S = len(sources), len(sources[0])
    res = []
    for v in range(V):
        for j, u in enumerate(sources[v]):
            locs = None if sample_locs_in is None else sample_locs_in[:, v, j].contiguous()
            res.append(epi.epipolar_fusion(feats[v], feats[u], P[v], P[u], sample_locs_in=locs, **kw))
    out = []
    for i, r in enumerate(zip(*res)):
        if r[0] is None:
            out.append(None)
            continue
        t = torch.stack(list(r)).unflatten(0, (V, S))
        out.append(t.permute(2, 0, 1, *range(3, t.dim())) if i == 3 else t)
    return out


def assert_equal(got, want, tag=""):
    for what, g, w in zip(OUTS, got, want):
        if w is None:
            assert g is None, what
            continue
        assert g.shape == w.shape and g.dtype == torch.float32, (tag, what, g.shape, w.shape)
        assert torch.equal(g, w), "%s %s differs: max |diff| %.3g" % (tag, what, (g - w).abs().max().item())


def assert_table_equals_singles(feats, P, sources, state=None, **kw):
    kw.setdefault("want_locs", True)
    want = singles(feats, P, sources, **kw)
    got = epi.epipolar_fusion_views(feats, P, state=state, sources=sources, **kw)
    torch.cuda.synchronize()
    assert_equal(got, want)
    return got


# ---- bit-exactness against V·S single calls --------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", TABLES)
@pytest.mark.parametrize("variant", ["auto", "pipe", "sector", "tile", "warp"])
@pytest.mark.parametrize("V", [2, 4, 5])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_pair_identity(dtype, V, variant, kind):
    if kind == "nobodys_source" and V == 2:
        pytest.skip("with two views each is the other's source")
    feats, P, kw = view_inputs(V, 2, 64, 32, 32, 32, seed=V)
    feats = feats.to(dtype)
    if not variant_supported(feats, P, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    assert_table_equals_singles(feats, P, table(kind, V), variant=variant, **kw)


@pytest.mark.parametrize("epilogue", ["add_ref", "z+zres", "z+zres+add_ref"])
@pytest.mark.parametrize("variant", ["auto", "warp"])
@pytest.mark.parametrize("C", [64, 264])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_epilogues(dtype, C, variant, epilogue):
    """residuals read the pair's query view feats[v][n]: the direct store, the transposition pass, the tensor-core z GEMM
    (C = 64) and the fp32 z epilogue (C = 264)"""
    feats, P, kw = view_inputs(4, 2, C, 16, 16, 16, seed=C)
    kw.update(add_ref_residual="add_ref" in epilogue, variant=variant)
    if epilogue.startswith("z"):
        kw.update(z_folded=random_z(C, C), z_residual=True)
    assert_table_equals_singles(feats.to(dtype), P, table("duplicates", 4), **kw)


@pytest.mark.parametrize("variant", ["auto", "tile", "warp"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_injected_sample_locs(dtype, variant):
    feats, P, kw = view_inputs(4, 2, 64, 24, 24, 16, seed=3)
    feats = feats.to(dtype)
    src = table("s2", 4)
    locs = epi.epipolar_fusion_views(feats, P, want_locs=True, sources=src, **kw)[3]          # [K,V,S,N,H,W,2]
    assert locs.shape[1:4] == (4, 2, 2)
    g = torch.Generator(device="cuda").manual_seed(4)
    locs = (locs + 0.02 * (torch.rand(locs.shape, device="cuda", generator=g) - 0.5)).contiguous()
    assert_table_equals_singles(feats, P, src, sample_locs_in=locs, variant=variant, want_locs=False, **kw)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_benchmark_shape(dtype):
    """the standard test's shape: four views, nearest camera, C = 256 on 64×64 maps (64-pixel items), K = 64, z + ZRESIDUAL and
    the caller residual"""
    feats, P, kw = view_inputs(4, 2, 256, 64, 64, 64, seed=9)
    kw.update(z_folded=random_z(256, 2), z_residual=True, add_ref_residual=True)
    src = multiview.nearest_view_table(P[:, 0])
    for variant in ("pipe", "auto"):
        assert_table_equals_singles(feats.to(dtype), P, src.tolist(), variant=variant, **kw)


# ---- the all-others table is the all-others form ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["auto", "sector", "tile", "warp"])
@pytest.mark.parametrize("V", [2, 4, 5])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_all_others_table_equals_views_form(dtype, V, variant):
    """sources = every other view in increasing order gives the bits of sources=None, in the same number of launches"""
    feats, P, kw = view_inputs(V, 2, 64, 32, 32, 32, seed=20 + V)
    feats = feats.to(dtype)
    if not variant_supported(feats, P, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    kw.update(variant=variant, want_locs=True, z_folded=random_z(64, V), z_residual=True, add_ref_residual=True)
    lib = _lib.load()
    want = epi.epipolar_fusion_views(feats, P, **kw)
    n_views = lib.epi_last_launch_count()
    got = epi.epipolar_fusion_views(feats, P, sources=np.array([others(V, v) for v in range(V)]), **kw)
    assert lib.epi_last_launch_count() == n_views
    assert_equal(got, want)


@pytest.mark.parametrize("variant", ["auto", "pipe", "sector", "tile", "warp"])
def test_launch_count(variant):
    """a table call launches what the views call launches"""
    feats, P, kw = view_inputs(4, 2, 64, 32, 32, 32, seed=4)
    if not variant_supported(feats, P, variant, **kw):
        pytest.skip("%s kernel does not take this shape" % variant)
    lib = _lib.load()
    for extra in ({}, dict(z_folded=random_z(64, 1), z_residual=True)):
        epi.epipolar_fusion_views(feats, P, variant=variant, **kw, **extra)
        n = lib.epi_last_launch_count()
        epi.epipolar_fusion_views(feats, P, variant=variant, sources=table("nearest", 4), **kw, **extra)
        assert lib.epi_last_launch_count() == n


# ---- the persistent cache --------------------------------------------------------------------------------------------------
def test_fusion_state_cache():
    """one FusionState through table and camera changes: every call equals fresh single calls"""
    V, N = 4, 2
    feats, P, kw = view_inputs(V, N, 64, 32, 32, 32, seed=6)
    kw.update(z_folded=random_z(64, 3), z_residual=True, variant="pipe")
    Pb = P.clone()
    Pb[2] = P[2].flip(0)
    st = epi.FusionState()
    for Pi, kind in ((P, "nearest"), (P, "nearest"), (P, "everybodys_source"), (Pb, "everybodys_source"), (P, "s2"),
                     (P, "nearest")):
        assert_table_equals_singles(feats, Pi, table(kind, V), state=st, **kw)


def _table_call(p, src, ws, cache):
    lib = _lib.load()
    t = np.ascontiguousarray(src, dtype=np.int32)
    tp = t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()
    p.cache, p.cache_bytes = (cache.data_ptr(), cache.numel()) if cache is not None else (None, 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.epi_fusion_view_sources_forward_f32(ctypes.byref(p), tp, t.shape[1], stream), "view sources forward")
    torch.cuda.synchronize()


def test_cache_keyed_by_pair_cameras():
    """one cache buffer, kept across calls whose tables differ (same V·S·N pairs): each pair's cached constants and orders are
    keyed by its own cameras, so every call equals a call without a cache"""
    V, N, C, H, W, K = 4, 2, 64, 32, 32, 32
    feats, P, _ = view_inputs(V, N, C, H, W, K, seed=7)
    f = feats.flatten(0, 1)
    NP = V * N
    lib = _lib.load()
    cache = None
    for kind in ("nearest", "everybodys_source", "nobodys_source", "nearest"):
        src = table(kind, V)
        res = []
        for use_cache in (True, False):
            out, attn = torch.empty(NP, C, H, W, device="cuda"), torch.empty(NP, K, H, W, device="cuda")
            p = fusion_params(f, f, out, K=K, P1=P.reshape(V * N, 3, 4), attn=attn, variant="pipe")
            p.N, p.n_views, p.feat_src, p.P_src = N, V, None, None
            t = np.ascontiguousarray(src, dtype=np.int32)
            targs = (t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 1)
            if use_cache and cache is None:
                cache = torch.zeros(lib.epi_fusion_view_sources_cache_bytes(ctypes.byref(p), *targs), device="cuda", dtype=torch.uint8)
            ws = torch.empty(lib.epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), *targs), device="cuda", dtype=torch.uint8)
            _table_call(p, src, ws, cache if use_cache else None)
            res.append((out, attn))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), kind


# ---- layouts and buffers ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["channels_last", "strided", "odd_13x19", "list_of_maps"])
def test_layouts(layout):
    V, N, C, H, W = 4, 2, 64, 32, 32
    if layout == "odd_13x19":
        H, W = 13, 19
    feats, P, kw = view_inputs(V, N, C, H, W, 16, seed=11)
    if layout == "channels_last":
        feats = feats.flatten(0, 1).contiguous(memory_format=torch.channels_last).unflatten(0, (V, N))
    elif layout == "strided":
        big = torch.zeros(V, N, 2 * C, H, W + 3, device="cuda")
        big[:, :, ::2, :, :W] = feats
        feats = big[:, :, ::2, :, :W]
    src = table("s2", V)
    for variant in ("auto", "warp"):
        want = singles(feats, P, src, variant=variant, want_locs=True, add_ref_residual=True, **kw)
        got = epi.epipolar_fusion_views(list(feats) if layout == "list_of_maps" else feats, P, variant=variant, want_locs=True,
                                        add_ref_residual=True, sources=src, **kw)
        assert_equal(got, want, variant)


@pytest.mark.parametrize("case", ["pipe_z", "pipe_unstage_bf16", "warp_f16", "sector"])
def test_outputs_written_and_workspace_independent(case):
    """outputs between NaN-pattern guards, the workspace prefilled with 0x00 and then 0xFF: every output element is written,
    no guard is, and both runs give the same bits as the single calls"""
    variant, dtype, z = {"pipe_z": ("pipe", torch.float32, True), "pipe_unstage_bf16": ("pipe", torch.bfloat16, False),
                         "warp_f16": ("warp", torch.float16, False), "sector": ("sector", torch.float32, False)}[case]
    V, N, C, H, W, K = 4, 2, 64, 32, 32, 32
    feats, P, kw = view_inputs(V, N, C, H, W, K, seed=12)
    feats = feats.to(dtype)
    zw = random_z(C, 5) if z else None
    src = table("duplicates", V)
    S = len(src[0])
    NP = V * S * N
    f = feats.flatten(0, 1)
    t = np.ascontiguousarray(src, dtype=np.int32)
    targs = (t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), S)
    runs = []
    for fill in (0x00, 0xFF):
        outs = dict(out=Guarded((NP, C, H, W)), attn=Guarded((NP, K, H, W)), corr=Guarded((NP, H, W, 2)),
                    locs=Guarded((K, NP, H, W, 2)))
        p = fusion_params(f, f, outs["out"].t, K=K, P1=P.reshape(V * N, 3, 4), attn=outs["attn"].t, corr=outs["corr"].t,
                          locs_out=outs["locs"].t, z=zw, z_residual=z, add_ref=True, variant=variant)
        p.N, p.n_views, p.feat_src, p.P_src = N, V, None, None
        nbytes = _lib.load().epi_fusion_view_sources_workspace_bytes(ctypes.byref(p), *targs)
        ws = poisoned(nbytes, fill)
        _table_call(p, src, ws, None)
        assert (ws[nbytes:] == fill).all(), "the guard behind the workspace was written"
        for k, g in outs.items():
            g.check("%s (workspace 0x%02X)" % (k, fill))
        runs.append({k: g.t.clone() for k, g in outs.items()})
    for k in runs[0]:
        assert torch.equal(int_bits(runs[0][k]), int_bits(runs[1][k])), "%s depends on the workspace's old contents" % k
    want = singles(feats, P, src, variant=variant, want_locs=True, add_ref_residual=True, z_folded=zw, z_residual=z, **kw)
    for k, w in zip(("out", "corr", "attn", "locs"), want):
        assert torch.equal(runs[0][k], w.flatten(1, 3) if k == "locs" else w.flatten(0, 2)), k


def test_inference_only_and_device_table():
    feats, P, kw = view_inputs(2, 1, 16, 12, 12, 8, seed=8)
    with pytest.raises(RuntimeError, match="epipolar_fusion"):
        epi.epipolar_fusion_views(feats.requires_grad_(True), P, sources=[[1], [0]], **kw)
    with torch.no_grad():
        with pytest.raises(TypeError, match="synchronise"):
            epi.epipolar_fusion_views(feats, P, sources=torch.tensor([[1], [0]], device="cuda"), **kw)
        epi.epipolar_fusion_views(feats, P, sources=torch.tensor([[1], [0]]), **kw)


# ---- the module and the test helpers ---------------------------------------------------------------------------------------
def _module(fuse_ref):
    cfg = epi.cfg_h36m_r50_256()
    cfg.VIS.EPIPOLAR_LINE = True
    m = epi.Epipolar(cfg=cfg, fuse_ref_residual=fuse_ref).cuda().eval()
    params = syn.z_bn_params(cfg.KEYPOINT.NFEATS, 5)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    return m, cfg


@pytest.mark.parametrize("fuse_ref", [False, True])
def test_forward_views_equals_forward_loop(fuse_ref):
    m, cfg = _module(fuse_ref)
    C, (H, W) = cfg.KEYPOINT.NFEATS, cfg.KEYPOINT.HEATMAP_SIZE
    V = 4
    feats, P, _ = view_inputs(V, 1, C, H, W, cfg.EPIPOLAR.SAMPLESIZE, seed=12)
    with torch.no_grad():
        for kind in ("nearest", "s2"):                              # one module state through a table change
            src = table(kind, V)
            want = [[m(feats[v], feats[u], P[v], P[u]) for u in src[v]] for v in range(V)]
            got = m.forward_views(feats, P, sources=src)
            for i, what in enumerate(("finalout", "corr_pos", "attn", "sample_locs")):
                w = torch.stack([torch.stack([x[i] for x in row]) for row in want])
                assert torch.equal(got[i], w), (kind, what)
    m.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        m.forward_views(feats, P, sources=table("nearest", V))


def _proxy(fuse_ref):
    d = mpjpe_proxy.build(seed=0)
    sampler = epi.Epipolar(cfg=d["cfg"], fuse_ref_residual=fuse_ref).cuda().eval()
    conv = torch.nn.Conv2d(mpjpe_proxy.C, mpjpe_proxy.J, 1, bias=False).cuda()
    conv.weight.data.copy_(torch.from_numpy(d["head"])[:, :, None, None])

    def tail(x):                                                # per item, so batch size cannot change the head's arithmetic
        return torch.cat([conv(x[i:i + 1]) for i in range(x.shape[0])])

    feats = dev(d["feat_ref"])[:, None]                         # [V,1,C,H,W]: view v of one frame
    KRT = dev(d["KRT"].astype(np.float32))
    return sampler, tail, feats, KRT[:, None], KRT


@pytest.mark.parametrize("fuse_ref", [False, True])
def test_standard_views_test_equals_two_pass_flow(fuse_ref):
    """one table call on one backbone pass equals the reference's standard test: per view, getOtherFeat on (view, its nearest
    camera's view), the tail, then the peak finder"""
    sampler, tail, feats, P, KRT = _proxy(fuse_ref)
    V = feats.shape[0]
    src = multiview.nearest_view_table(KRT, topk=1)
    sigma, ds = 2.0, 4.0
    locs, scores, corr, attn = epi.standard_views_test(sampler, tail, feats, P, src, sigma, ds)
    assert locs.shape[:2] == scores.shape[:2] == (V, 1)
    with torch.no_grad():
        for v in range(V):
            u = int(src[v, 0])
            ret, c, a, _ = epi.fused_other_feat(feats[v], feats[u], P[v], P[u], sampler)
            wl, ws = epi.find_tensor_peak_batch(tail(ret), sigma, ds)
            assert torch.equal(locs[v], wl) and torch.equal(scores[v], ws), v
            assert torch.equal(corr[v], c) and torch.equal(attn[v], a), v


@pytest.mark.parametrize("fuse_ref", [False, True])
def test_multitest_views_k_nearest(fuse_ref):
    """multitest over each view's two nearest cameras equals `multitest` run per view over those sources, with the winner
    reported as its camera index"""
    sampler, tail, feats, P, KRT = _proxy(fuse_ref)
    V = feats.shape[0]
    src = multiview.nearest_view_table(KRT, topk=2)
    sigma, ds = 2.0, 4.0
    locs, scores, cam = epi.multitest_views(sampler, tail, feats, P, sigma, ds, sources=src)
    for v in range(V):
        us = [int(u) for u in src[v]]
        wl, ws, wj = epi.multitest(sampler, tail, feats[v], feats[us], P[v], P[us], sigma, ds)
        assert torch.equal(locs[v], wl) and torch.equal(scores[v], ws), v
        assert torch.equal(cam[v], torch.tensor(us, device=wj.device)[wj]), v
