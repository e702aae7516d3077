"""GPU: the peak finders (csrc/epi_peaks.cu) at the edges: the reference's own outputs on non-finite, tied and degenerate maps
(tests/golden/peaks_edges.npz), a sweep against the numpy oracle in fp64, batching, input dtypes and layouts, the best-source
selection against torch.max over the oracle's peaks, and a NaN map's hand-off to triangulation.

Non-finite values follow torch: a map holding a NaN scores its first NaN and, through the window's bilinear samples, has a
NaN location; the best source is the first one with a NaN score, else the first highest score."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from oracle import make_golden_peaks as mg
from oracle import mpjpe_proxy, peaks_oracle as po, triangulate_oracle as to
from tests.test_peaks_edges_cpu import assert_matches_golden

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def oracle(heat, *args, **kw):
    with np.errstate(invalid="ignore"):                                 # 0 · inf and inf - inf in the non-finite cases
        return po.find_tensor_peak_batch(heat, *args, **kw)


# ---- the reference's outputs -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(mg.EDGES))
def test_kernel_matches_reference_golden(name):
    J, H, W, radius, ds, _ = mg.EDGES[name]
    h = dev(mg.edge_heatmaps(name))
    locs, score = epi.find_tensor_peak_batch(h, radius, ds)
    assert_matches_golden(name, locs.cpu().numpy(), score.cpu().numpy())
    # the best-source kernel over two copies of the map: the first source, and the single-source bits
    bl, bs, src = epi.find_tensor_peak_best(torch.stack([h, h])[:, None], radius, ds)
    assert same_bits(bl[0], locs) and same_bits(bs[0], score) and (src == 0).all()


# ---- sweep against the fp64 oracle -------------------------------------------------------------------------------------------
def sweep_maps(kind, B, J, H, W, seed):
    """pos: a bump on non-negative noise; ties: noise < 0.5 with 2 to 4 pixels at exactly 1.0, in any lanes; signed: a bump on
    zero-mean noise, so that a negative threshold keeps samples of both signs"""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.empty((B, J, H, W), np.float32)
    for b in range(B):
        for j in range(J):
            cx, cy, sg = rng.uniform(-1, W), rng.uniform(-1, H), rng.uniform(1.0, 3.0)
            g = np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * sg ** 2))
            if kind == "pos":
                m = g + 0.3 * rng.random((H, W))
            elif kind == "ties":
                m = 0.5 * rng.random((H, W))
                m.reshape(-1)[rng.choice(H * W, size=rng.integers(2, 5), replace=False)] = 1.0
            else:
                m = 1.5 * g + 0.8 * rng.standard_normal((H, W))
            out[b, j] = m.astype(np.float32)
    return out


SHAPES = {"h36m": (2, 17, 64, 64, 8.0, 4.0), "odd": (3, 7, 13, 37, 2.6, 1.0)}    # B, J, H, W, radius, downsample
CANCEL = 512


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("int_div", [0, 1])
@pytest.mark.parametrize("threshold", [0.0, -1.0, 0.5])
@pytest.mark.parametrize("kind", ["pos", "ties", "signed"])
def test_sweep_against_fp64_oracle(kind, threshold, int_div, shape):
    """Scores are the map's values at the same arg-max, bit for bit.  Locations: where every kept sample has one sign, within
    3e-4·(downsample/4) image px of the oracle in fp64.  A signed map under a negative threshold keeps samples of both signs,
    and Σ sub can nearly cancel; there the float32 sums and the rounded bilinear weights, whose coordinates reach max(H, W),
    move the centroid by up to CANCEL·2^-24·Σ|sub|·(radius + 1)/|Σ sub| feature px on top, times downsample in image px.
    The oracle's own float32 restatement needs a factor below 80 in place of CANCEL on these maps."""
    B, J, H, W, radius, ds = SHAPES[shape]
    heat = sweep_maps(kind, B, J, H, W, seed=len(kind) * 7 + int_div)
    locs, score = epi.find_tensor_peak_batch(dev(heat), radius, ds, threshold=threshold, int_div=bool(int_div))
    locs, score = locs.cpu().numpy(), score.cpu().numpy()
    for b in range(B):
        lo, so, sub = oracle(heat[b], radius, ds, threshold, int_div, dtype=np.float64, window=True)
        np.testing.assert_array_equal(score[b], so.astype(np.float32))
        tol = np.full(J, 3e-4 * ds / 4)
        if kind == "signed" and threshold < 0:
            flat = sub.reshape(J, -1)
            tol += CANCEL * U * np.abs(flat).sum(1) * (radius + 1) / np.abs(flat.sum(1)) * ds
        err = np.abs(locs[b] - lo).max(1)
        assert (err <= tol).all(), (b, err.max(), tol[err.argmax()])


# ---- batching, dtypes and layouts --------------------------------------------------------------------------------------------
def batch_maps():
    """[8, 2048, 8, 8]: 16384 warps, 4096 blocks; a NaN in every 97th map and -inf in every 89th"""
    g = torch.Generator(device="cuda").manual_seed(3)
    h = torch.rand(8, 2048, 8, 8, device="cuda", generator=g)
    f = h.view(-1, 64)
    f[::97, 13] = float("nan")
    f[::89, 40] = float("-inf")
    return h


def test_batched_equals_per_item():
    h = batch_maps()
    locs, score = epi.find_tensor_peak_batch(h, 2.0, 4.0)
    assert torch.isnan(score).any() and torch.isnan(locs).any()
    for b in range(h.shape[0]):
        li, si = epi.find_tensor_peak_batch(h[b], 2.0, 4.0)
        assert same_bits(locs[b], li) and same_bits(score[b], si), b
    lb, sb, src = epi.find_tensor_peak_best(h[None], 2.0, 4.0)
    assert same_bits(lb, locs) and same_bits(sb, score) and (src == 0).all()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_half_heat_gives_its_fp32_copy(dtype):
    """half-precision heat is widened to fp32 exactly and the peak is computed in fp32"""
    h = batch_maps()[:2].to(dtype)
    for args in ((2.0, 4.0), (2.6, 8.0, -1.0, True)):
        a = epi.find_tensor_peak_batch(h, *args)
        b = epi.find_tensor_peak_batch(h.float(), *args)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    a = epi.find_tensor_peak_best(torch.stack([h, h.flip(1)]), 2.0, 4.0)
    b = epi.find_tensor_peak_best(torch.stack([h, h.flip(1)]).float(), 2.0, 4.0)
    assert all(same_bits(x, y) for x, y in zip(a, b))


def test_strided_and_channels_last_heat():
    g = torch.Generator(device="cuda").manual_seed(4)
    big = torch.randn(3, 10, 21, 30, device="cuda", generator=g)
    big[1, 4, 5, 6] = float("nan")
    for h in (big.contiguous(memory_format=torch.channels_last), big[:, ::2, 1:-2, 3:], big.transpose(2, 3)):
        a = epi.find_tensor_peak_batch(h, 3.0, 4.0, threshold=-0.5)
        b = epi.find_tensor_peak_batch(h.contiguous(), 3.0, 4.0, threshold=-0.5)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
        a = epi.find_tensor_peak_best(torch.stack([h, h * 2]), 3.0, 4.0)
        b = epi.find_tensor_peak_best(torch.stack([h, h * 2]).contiguous(), 3.0, 4.0)
        assert all(same_bits(x, y) for x, y in zip(a, b))


# ---- best source against torch.max over the oracle's peaks -------------------------------------------------------------------
def oracle_best(heat, radius, ds):
    """modeling/model.py:229-234 over the oracle: torch.max over the sources' scores (first NaN, else first maximum), gather"""
    S, B = heat.shape[:2]
    res = [[oracle(heat[s, b], radius, ds) for b in range(B)] for s in range(S)]
    locs = np.stack([[r[0] for r in row] for row in res])                  # [S,B,J,2]
    scores = torch.from_numpy(np.stack([[r[1] for r in row] for row in res]))
    best, idx = torch.max(scores, 0)
    return np.take_along_axis(locs, idx.numpy()[None, ..., None], 0)[0], best.numpy(), idx.numpy()


def best_source_maps(S, seed):
    """[S, 2, 7, 16, 20]; joint j of every frame is one case (BEST_CASES[j])"""
    B, J, H, W = 2, len(BEST_CASES), 16, 20
    rng = np.random.default_rng(seed)
    heat = rng.random((S, B, J, H, W)).astype(np.float32)
    last, mid = S - 1, S // 2
    for b in range(B):
        heat[last, b, 0, 3 + b, 4] = np.nan                                 # NaN in a later source
        heat[[max(0, last - 1), last], b, 1, 7, 2 + b] = np.nan             # NaN in two sources: the first of them
        heat[0, b, 2, 5, 5] = np.inf                                        # +inf in the first source, NaN in the last
        heat[last, b, 2, 9, 1] = np.nan
        heat[:, b, 3] = -np.inf                                             # all -inf everywhere
        heat[:, b, 4] = heat[0, b, 4]                                       # exact ties: every source the same map
        heat[0, b, 5] *= 0.5                                                # ties between the later sources only
        heat[1:, b, 5] = heat[min(1, last), b, 5]
        heat[[mid, last], b, 6, 2, 3 + b] = np.inf                          # +inf in two sources: the first of them
    return heat


BEST_CASES = ["NaN in a later source", "NaN in two sources", "NaN against +inf", "all -inf", "every source tied",
              "later sources tied", "+inf in two sources"]


@pytest.mark.parametrize("S", [1, 2, 3, 8])
def test_best_source_against_oracle(S):
    heat = best_source_maps(S, seed=S)
    radius, ds = 2.0, 4.0
    locs, scores, src = epi.find_tensor_peak_best(dev(heat), radius, ds)
    wl, ws, wi = oracle_best(heat, radius, ds)
    locs, scores, src = locs.cpu().numpy(), scores.cpu().numpy(), src.cpu().numpy()
    for j, case in enumerate(BEST_CASES):
        np.testing.assert_array_equal(src[:, j], wi[:, j], err_msg=case)
        np.testing.assert_array_equal(scores[:, j].view(np.uint32), ws[:, j].view(np.uint32), err_msg=case)
        np.testing.assert_array_equal(np.isnan(locs[:, j]), np.isnan(wl[:, j]), err_msg=case)
        np.testing.assert_allclose(locs[:, j], wl[:, j], rtol=0, atol=3e-4, equal_nan=True, err_msg=case)
    if S >= 2:
        assert (src[:, 0] == S - 1).all() and (src[:, 1] == S - 2).all() and (src[:, 2] == S - 1).all()
        assert np.isnan(scores[:, :3]).all()
    assert (src[:, 3:5] == 0).all() and (src[:, 5] == min(1, S - 1)).all() and (src[:, 6] == S // 2).all()


def test_best_source_without_src_index():
    """src_index = NULL through the C ABI: the same locations and scores"""
    h = dev(best_source_maps(3, seed=9))
    locs, scores, _ = epi.find_tensor_peak_best(h, 2.0, 4.0)
    S, B, J, H, W = h.shape
    l2, s2 = torch.full_like(locs, 7.0), torch.full_like(scores, 7.0)
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.epi_find_peaks_best_f32(h.data_ptr(), l2.data_ptr(), s2.data_ptr(), None, S, B, J, H, W, 2.0, 4.0, 1e-6, 0,
                                           ctypes.c_void_p(stream)), "epi_find_peaks_best_f32")
    torch.cuda.synchronize()
    assert same_bits(l2, locs) and same_bits(s2, scores)


# ---- hand-off to triangulation -----------------------------------------------------------------------------------------------
def test_nan_map_is_dropped_by_triangulation():
    """The MPJPE proxy scene's heat (its 1x1 head over each view's features) with a NaN in one (view, joint) map:
    find_tensor_peak_batch -> triangulate_views agrees with peaks_oracle -> triangulate_oracle.  The poisoned view scores NaN,
    so it is not selected for that joint, which still triangulates from the other views; every other joint keeps its bits."""
    d = mpjpe_proxy.build(0)
    V, J = mpjpe_proxy.V, mpjpe_proxy.J
    heat = np.einsum("jc,vchw->vjhw", d["head"].astype(np.float64), d["feat_ref"].astype(np.float64)).astype(np.float32)
    P = d["KRT"][:, None]                                                   # [V,1,3,4] fp64
    pv, pj = 1, 5
    bad = heat.copy()
    bad[pv, pj, 0, 0] = np.nan                                              # far from the joint's peak

    def gpu(h):
        locs, scores = epi.find_tensor_peak_batch(dev(h), 2.0, 4.0)
        X, n = epi.triangulate_views(locs[:, None], scores[:, None], dev(P))
        return X[0], n[0], scores

    def host(h):
        lo, so = zip(*[oracle(h[v], 2.0, 4.0) for v in range(V)])
        X, n, _ = to.triangulate(np.stack(lo)[:, None], np.stack(so)[:, None], P)
        return X[0], n[0]

    X0, n0, _ = gpu(heat)
    X, n, scores = gpu(bad)
    Xo, no = host(bad)
    assert torch.isnan(scores[pv, pj]) and torch.isfinite(scores[:, :pj]).all()
    n = n.cpu().numpy()
    np.testing.assert_array_equal(n, no)
    assert n[pj] == V - 1 and (np.delete(n, pj) == V).all() and (n0 == V).all()
    X, X0 = X.cpu().numpy(), X0.cpu().numpy()
    assert np.isfinite(X).all()
    assert np.linalg.norm(X - Xo, axis=-1).max() <= 0.01                    # mm: 3e-4 px of 2-D agreement moves a ray by < 0.01 mm
    keep = np.arange(J) != pj
    np.testing.assert_array_equal(X[keep], X0[keep])
    assert np.linalg.norm(X[pj] - d["joints"][pj]) < 30.0                  # mm: three views still find the joint
