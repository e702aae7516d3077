"""GPU: triangulate_views (csrc/epi_triangulate.cu) against the numpy oracle (oracle/triangulate_oracle.py) on >= 1e5 problems,
on the MPJPE proxy scene and behind the real eval chain, without a host sync, in a CUDA graph, and against producers on the
current and on a side stream."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, multiview, synthetic as syn
from oracle import mpjpe_proxy, triangulate_oracle as to
from tests.test_gpu_view_sources import _proxy

pytestmark = pytest.mark.gpu
J = 17
# scores spread over several 0.05 bins, across -1 and below it, with NaN and the exact float32 threshold
SCORE_BINS = np.array([0.9, 0.3, 0.06, 0.05, 0.04, 0.0, -0.03, -0.2, -0.55, -0.98, -1.0, -1.04, -2.0, np.nan])


def lookat_rig(rng, V):
    """V cameras at random distances (2-8 m) and directions, looking near the origin, random focal lengths and centres"""
    out = np.zeros((V, 3, 4))
    for v in range(V):
        f = rng.uniform(200, 2000)
        K = np.array([[f, 0, rng.uniform(100, 600)], [0, f * rng.uniform(0.9, 1.1), rng.uniform(100, 600)], [0, 0, 1]])
        C = rng.standard_normal(3)
        C *= rng.uniform(2000, 8000) / np.linalg.norm(C)
        z = rng.normal(0, 300, 3) - C
        z /= np.linalg.norm(z)
        x = np.cross(z, rng.standard_normal(3))
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        out[v] = K @ np.concatenate([R, -R @ C[:, None]], 1)
    return out


def scene(kind, V, N, seed):
    """locs [V,N,J,2] float32, scores [V,N,J] float32, P [V,N,3,4] float64: joints projected through each frame's rig, jittered"""
    rng = np.random.default_rng(seed)
    if kind == "ring":
        P = np.stack([syn.ring_cameras(V, 256, jitter=30.0, seed=seed * 1000 + n) for n in range(N)], 1)
        X = np.array([0.0, 0.0, 1000.0]) + rng.uniform(-600, 600, (N, J, 3))
    elif kind == "lookat":
        P = np.stack([lookat_rig(rng, V) for _ in range(N)], 1)
        X = rng.normal(0, 400, (N, J, 3))
    else:                                                                       # literal randn cameras (syn.random_krt)
        P = rng.standard_normal((V, N, 3, 4))
        X = rng.standard_normal((N, J, 3))
    Xh = np.concatenate([X, np.ones((N, J, 1))], -1)
    uv = np.einsum("vnrc,njc->vnjr", P, Xh)
    locs = uv[..., :2] / uv[..., 2:3]
    locs += rng.normal(0, 1.0 if kind != "randn" else 1e-3, locs.shape)
    scores = rng.choice(SCORE_BINS, (V, N, J)) + np.where(rng.random((V, N, J)) < 0.5, 0, rng.uniform(-0.01, 0.01, (V, N, J)))
    return locs.astype(np.float32), scores.astype(np.float32), P


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def exact_dlt(locs, scores, P, conf, n, j):
    """X of problem (n, j) from A's null vector in 40-digit arithmetic (mpmath ships with torch's sympy)"""
    import mpmath
    mpmath.mp.dps = 40
    sel = np.flatnonzero(to.selection_mask(scores[:, n, j][:, None], conf)[:, 0])
    A = []
    for v in sel:
        M = P[v, n].astype(np.float64)
        A += [np.float64(locs[v, n, j, 0]) * M[2] - M[0], np.float64(locs[v, n, j, 1]) * M[2] - M[1]]
    A = mpmath.matrix(np.stack(A).tolist())
    E, Q = mpmath.eigsy(A.T * A)
    k = min(range(4), key=lambda i: E[i])
    return np.array([float(Q[i, k] / Q[3, k]) for i in range(3)])


def compare(kind, locs, scores, P, Pdev, conf=0.05):
    """Where the kernel is farther from the oracle than the bound, the oracle's own fp64 error can be the cause: numpy's SVD
    of a two-view A whose rays nearly meet at a distant point (|X| ~ 300 m on a ring) is off by ~5e-6 mm.  Such a problem
    passes when the kernel is within the bound of A's null vector in 40-digit arithmetic and closer to it than the oracle."""
    X, n = epi.triangulate_views(dev(locs), dev(scores), Pdev, conf)
    X, n = X.cpu().numpy(), n.cpu().numpy()
    Pn = Pdev.cpu().numpy()
    Xo, no, sv = to.triangulate(locs, scores, Pn, conf)
    assert (n == no).all(), "n_used differs at %d problems" % (n != no).sum()
    assert (np.isnan(X) == np.isnan(Xo)).all()
    ok = ~np.isnan(Xo).any(-1)
    err = np.where(ok, np.linalg.norm(X - Xo, axis=-1), 0.0)
    if kind == "ring":
        bound = np.full(err.shape, 1e-6)
    else:
        gap = sv[..., 2] >= 2 * sv[..., 3]
        assert gap[ok].mean() > 0.5
        bound = np.where(gap, 1e-9 * np.linalg.norm(Xo, axis=-1), np.inf)
    over = np.argwhere(ok & (err > bound))
    assert len(over) <= 1e-3 * ok.sum(), "%d problems over the bound" % len(over)
    for nn, j in over:
        Xe = exact_dlt(locs, scores, Pn, conf, nn, j)
        ek, eo = np.linalg.norm(X[nn, j] - Xe), np.linalg.norm(Xo[nn, j] - Xe)
        assert ek <= bound[nn, j] and ek < eo, (kind, nn, j, err[nn, j], ek, eo)
    print("%s V=%d: max |dX| %.3g, %d problems where the oracle is the farther one from the 40-digit X"
          % (kind, P.shape[0], err.max(), len(over)))
    return ok.size, np.bincount(no.ravel(), minlength=P.shape[0] + 1)


@pytest.mark.parametrize("p_dtype", ["f64", "f32"])
def test_parity_with_oracle(p_dtype):
    """>= 1e5 problems: identical counts and NaN positions; |dX| <= 1e-6 mm on ring rigs, <= 1e-9·|X| on random rigs where the
    oracle's two smallest singular values differ by 2x or more"""
    total, counts = 0, []
    for kind, V, N, seed in [("ring", 2, 800, 1), ("ring", 3, 800, 2), ("ring", 4, 1800, 3), ("ring", 8, 600, 4), ("ring", 64, 150, 5),
                             ("lookat", 2, 400, 6), ("lookat", 4, 400, 7), ("lookat", 8, 200, 8), ("randn", 3, 400, 9),
                             ("randn", 5, 400, 10)]:
        locs, scores, P = scene(kind, V, N, seed)
        Pdev = dev(P) if p_dtype == "f64" else dev(P.astype(np.float32))
        n, c = compare(kind, locs, scores, P, Pdev)
        total += n
        counts.append(c)
    assert total >= 10 ** 5
    # every count from 0 to 4 views occurs, so the relaxation, the final pass and the NaN rule are all exercised
    assert all(sum(c[k] for c in counts if len(c) > k) > 0 for k in range(5))


def test_nonfinite_inputs_give_nan():
    locs, scores, P = scene("ring", 4, 8, 11)
    scores[:] = 1.0
    locs[1, 0, 3, 0] = np.nan
    locs[2, 1, 5, 1] = np.inf
    P = P.copy()
    P[3, 2, 1, 2] = np.nan                                                      # every joint of frame 2
    scores[1, 3, 7] = np.nan                                                    # view 1 of (3, 7) not selected: still finite
    locs[1, 3, 7] = np.nan
    X, n = epi.triangulate_views(dev(locs), dev(scores), dev(P))
    X, n = X.cpu().numpy(), n.cpu().numpy()
    bad = np.zeros((8, J), bool)
    bad[0, 3] = bad[1, 5] = True
    bad[2] = True
    assert (np.isnan(X).any(-1) == bad).all() and (np.isnan(X).all(-1) == bad).all()
    assert n[3, 7] == 3 and (n[~bad] >= 3).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mpjpe_proxy_scene(seed, monkeypatch):
    """the layer's output through the proxy's head and peaks; every view used (scores above conf_thres): the joints match the
    proxy's numpy DLT to 1e-6 mm, and so does the MPJPE.  The proxy's 2-D points are rounded to float32 (what the kernel reads)
    before its DLT runs on them."""
    d = mpjpe_proxy.build(seed)
    out, _, _, _ = epi.epipolar_fusion(dev(d["feat_ref"]), dev(d["feat_src"]), dev(d["P_ref"]), dev(d["P_src"]), K=mpjpe_proxy.K,
                                       correct_normalize=True)
    fused = out.cpu().numpy()
    seen = []
    peaks = mpjpe_proxy._peaks

    def peaks_f32(heat):                                                        # image px = p·4 + 2 - 0.5, exact in fp64
        img = (peaks(heat) * 4.0 + 1.5).astype(np.float32).astype(np.float64)
        seen.append(img)
        return (img - 1.5) / 4.0

    monkeypatch.setattr(mpjpe_proxy, "_peaks", peaks_f32)
    want = mpjpe_proxy.mpjpe(d, fused)
    V = mpjpe_proxy.V
    locs = np.stack(seen).astype(np.float32)[:, None]                           # [V,1,J,2]
    P = d["KRT"][:, None]
    X, n = epi.triangulate_views(dev(locs), torch.ones(V, 1, J, device="cuda"), dev(P), conf_thres=0.05)
    X, n = X[0].cpu().numpy(), n.cpu().numpy()
    assert (n == V).all()
    Xo = to.triangulate(locs, np.ones((V, 1, J), np.float32), P)[0][0]
    assert np.linalg.norm(X - Xo, axis=-1).max() <= 1e-6
    got = float(np.mean(np.linalg.norm(X - d["joints"], axis=-1)))
    assert abs(got - want) <= 1e-6, (got, want)


def chain(sampler, conv, feats, P, src, fuse_head):
    locs, scores, _, _ = epi.standard_views_test(sampler, conv, feats, P, src, 2.0, 4.0, fuse_head=fuse_head)
    return epi.triangulate_views(locs, scores, P)


def test_real_chain_fused_head_mpjpe():
    """standard_views_test(fuse_head=True) -> triangulate_views on the proxy scene: the MPJPE of the unfused path, within what
    the 2-D peaks' 1e-3 px agreement allows (|dX| <= 0.05 mm: 1e-3 px at about 5 m and f = 290 px moves a ray by about 0.02 mm)"""
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):          # the unfused tail in fp32, as the fused head
        sampler, tail, feats, P, KRT = _proxy(False)
        conv = next(c.cell_contents for c in tail.__closure__ if isinstance(c.cell_contents, torch.nn.Conv2d))
        src = multiview.nearest_view_table(KRT, topk=1)
        la = epi.standard_views_test(sampler, conv, feats, P, src, 2.0, 4.0)[0]
        lb = epi.standard_views_test(sampler, conv, feats, P, src, 2.0, 4.0, fuse_head=True)[0]
        assert (la - lb).abs().max().item() <= 1e-3
        Xa, na = chain(sampler, conv, feats, P, src, False)
        Xb, nb = chain(sampler, conv, feats, P, src, True)
    joints = torch.from_numpy(mpjpe_proxy.build(0)["joints"]).cuda()
    assert torch.equal(na, nb) and (na == feats.shape[0]).all()
    assert (Xa - Xb).norm(dim=-1).max().item() <= 0.05
    ea, eb = (Xa[0] - joints).norm(dim=-1).mean().item(), (Xb[0] - joints).norm(dim=-1).mean().item()
    print("MPJPE unfused %.6f mm, fused head %.6f mm" % (ea, eb))
    assert abs(ea - eb) <= 0.05 and ea < 30.0


def test_no_host_sync():
    locs, scores, P = scene("ring", 4, 64, 12)
    l, s, p = dev(locs), dev(scores), dev(P.astype(np.float32))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        X, n = epi.triangulate_views(l, s, p)
        X2, n2 = epi.triangulate_views(l.half(), s.bfloat16(), p.double())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(X).any() and n.shape == (64, J) and X2.dtype == torch.float64


def test_cuda_graph_chain():
    """the eval chain (fused-head standard test, peaks, triangulation) captured in one graph after a warm-up: replays on new
    maps equal eager calls bit for bit"""
    sampler, tail, feats, P, KRT = _proxy(False)
    conv = next(c.cell_contents for c in tail.__closure__ if isinstance(c.cell_contents, torch.nn.Conv2d))
    src = multiview.nearest_view_table(KRT, topk=1)
    maps = [feats.clone()] + [dev(mpjpe_proxy.build(s)["feat_ref"])[:, None] for s in (1, 2)]
    static = maps[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        chain(sampler, conv, static, P, src, True)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = chain(sampler, conv, static, P, src, True)
    for m in maps[1:] + maps[:1]:
        static.copy_(m)
        g.replay()
        want = chain(sampler, conv, m, P, src, True)
        torch.cuda.synchronize()
        assert torch.equal(out[1], want[1])
        assert torch.equal(out[0].nan_to_num(7.0), want[0].nan_to_num(7.0)) and torch.isfinite(want[0]).all()
    assert not torch.equal(chain(sampler, conv, maps[1], P, src, True)[0], chain(sampler, conv, maps[2], P, src, True)[0])


def test_producers_on_current_and_side_stream():
    """a sleep, then a copy that writes input set Y into locs, then the call with no synchronise: the result is eager(Y), on
    the current stream and with the producer on a side stream the current stream waits for"""
    a, b = scene("ring", 4, 256, 13), scene("ring", 4, 256, 14)
    s, P = dev(a[1]), dev(a[2])
    la, lb = dev(a[0]), dev(b[0])
    want = epi.triangulate_views(lb, s, P)
    other = epi.triangulate_views(la, s, P)
    torch.cuda.synchronize()
    assert not torch.equal(want[0].nan_to_num(0), other[0].nan_to_num(0))
    side = torch.cuda.Stream()
    for producer in ("current", "side"):
        x = la.clone()
        torch.cuda.synchronize()
        if producer == "current":
            torch.cuda._sleep(50_000_000)
            x.copy_(lb)
        else:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(50_000_000)
                x.copy_(lb)
            torch.cuda.current_stream().wait_stream(side)
        got = epi.triangulate_views(x, s, P)
        torch.cuda.synchronize()
        assert torch.equal(got[1], want[1]) and torch.equal(got[0].nan_to_num(7.0), want[0].nan_to_num(7.0)), producer


@pytest.mark.parametrize("poison", [float("nan"), 12345.0])
def test_poisoned_outputs_fully_overwritten(poison):
    """X and n_used prefilled with poison through the C ABI: every element is written (a NaN X only where the oracle has one)"""
    locs, scores, P = scene("ring", 5, 333, 15)
    lib = _lib.load()
    l, s, p = dev(locs), dev(scores), dev(P)
    X = torch.full((333, J, 3), poison, device="cuda", dtype=torch.float64)
    n = torch.full((333, J), -7, device="cuda", dtype=torch.int32)
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.epi_triangulate_dlt_f64(l.data_ptr(), s.data_ptr(), p.data_ptr(), _lib.EPI_DTYPE_F64, 0.05, 5, 333, J,
                                           X.data_ptr(), n.data_ptr(), ctypes.c_void_p(stream)), "epi_triangulate_dlt_f64")
    Xw, nw = epi.triangulate_views(l, s, p)
    torch.cuda.synchronize()
    assert torch.equal(n, nw) and (n >= 0).all()
    assert torch.equal(X.isnan(), Xw.isnan()) and torch.equal(X.nan_to_num(0.0), Xw.nan_to_num(0.0))
    Xo, no, _ = to.triangulate(locs, scores, P)
    assert (np.isnan(Xo) == X.isnan().cpu().numpy()).all()
