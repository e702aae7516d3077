"""GPU: every forward kernel on camera rigs whose epipoles lie inside the maps (tests/util.py::pair_rig): the ring's opposite
views, facing cameras (e1 on a pixel centre, or between pixels, or at the centre the staging order key measures from), a
source camera behind the reference camera, and rig90, whose pixel column 32 has rays parallel to the source image plane
(zz == 0 exactly in fp32), with its near-degenerate twin.

  T2  the emitted sample_locs against the reference's pinv geometry in fp64, on every pixel at least 0.5 feature px from e1:
      the same far set, and each sample within max(1e-3 px, the reference module's own fp32 error at that sample) (1e-3 px
      on the facing rig, where the reference raises).  The largest error and its distance from e1 are printed.
  degenerate pixel (its ray meets the source camera centre, so its line is undefined): the far sentinel, or K finite samples
      on one line through e2 from border to border of the pixel-centre rectangle.
  T3  every pixel: out and attn within 1e-4 of the C oracle on the emitted locations, attention rows summing to 1, corr_pos
      the first maximum of the fp64 attention (near-ties excepted, tests/util.py::check_corr), far pixels with uniform
      attention and out = 0 (or the residual).  A pixel one of whose fp64 scores lies within 3e-5 of 0 is left out of the
      out / attn / corr_pos comparisons: an fp32 sum there may cancel to exactly 0, which the reference's sim == 0 mask
      turns into a masked sample, in any summation order.
Also the views form and a source table on the ring's opposite views (and the benchmark's shape with z), and the backward
deriving its own geometry from the cameras."""
import functools

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward
from oracle import c_oracle, epipolar_oracle as eo, torch_port
from tests.test_gpu_backward import reference_grads, torch_reference
from tests.test_gpu_pipe_items import force_items32
from tests.test_gpu_views import random_z
from tests.util import (FAR_LOC, PAIR_RIGS, RIG_HW, check_corr, e1_distance, epipoles, img2feat, loc2feat, pair_rig,
                        rel_max, ring_opposite, rig_cfg)

pytestmark = pytest.mark.gpu
H = W = RIG_HW
C, K = 64, 64
TOL = 1e-4
SCALE = float(epi.make_cfg().EPIPOLAR.SOFTMAXSCALE)
RIGS = ["ring_opposite"] + PAIR_RIGS
DEGENERATE = {"facing": (32, 32), "behind": (32, 32)}
VARIANTS = ["pipe", "pipe32", "sector", "tile", "warp", "auto"]
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def geometry(name, P1b, P2b, n):
    """fp64 reference locations [K,n,H,W,2], the reference module's own per-sample error in feature px [K,n,H,W] (inf where it
    has no line or raises) and e1's distance [n,H,W] — for the pair cameras given as bytes."""
    P1 = np.frombuffer(P1b, np.float32).reshape(n, 3, 4).copy(); P2 = np.frombuffer(P2b, np.float32).reshape(n, 3, 4).copy()
    cfg = rig_cfg(K)
    ref = eo.sample_locs(cfg, P1, P2, H, W, K, np.float64, "reference")
    terr = np.full(ref.shape[:-1], np.inf)
    if name != "facing":
        tg = torch_port.TorchGeometry(cfg, H, W)(torch.from_numpy(P1), torch.from_numpy(P2)).numpy()
        both = (np.abs(tg).max(-1) < 50) & (np.abs(ref).max(-1) < 50)
        terr = np.where(both, np.abs(loc2feat(tg, H, W) - loc2feat(ref, H, W)).max(-1), np.inf)
    return ref, terr, e1_distance(P1, P2, H, W)


def inputs(N, dtype, seed=0):
    f1 = syn.features(N, C, H, W, "randn", seed + 1); f2 = syn.features(N, C, H, W, "randn", seed + 2)
    t1, t2 = dev(f1).to(dtype), dev(f2).to(dtype)
    return t1, t2, t1.float().cpu().numpy(), t2.float().cpu().numpy()      # the kernels compute on the exact map values


def fp64_attention(f1, f2, locs):
    """attn [N,K,H·W] in fp64 (the reference's op sequence through torch_reference) on the fp32 locations [K,N,H,W,2], and
    the pixels [N,H,W] one of whose fp64 scores lies within 3e-5 of 0: there an fp32 sum may cancel to exactly 0, which the
    reference's `sim[sim==0] = -1e10` masks, so that pixel's attention is ill-posed in fp32."""
    g = np.where(np.isfinite(locs).all(-1, keepdims=True), locs, FAR_LOC).astype(np.float64)
    N = g.shape[1]
    with torch.no_grad():
        t1, t2, tg = dev(f1).double(), dev(f2).double(), dev(g)
        _, a = torch_reference(t1, t2, t2, tg, SCALE)
        near0 = []
        for n in range(N):
            s = torch.nn.functional.grid_sample(t2[n:n + 1], tg[:, n].reshape(1, K * H, W, 2), align_corners=False)
            sim = (s.view(-1, K, H, W) * t1[n].unsqueeze(1)).sum(0)
            near0.append(((sim.abs() < 3e-5) & (sim != 0)).any(0).cpu().numpy())
    return a.reshape(N, K, H * W).cpu().numpy(), np.stack(near0)


def check_t2(name, P1, P2, locs, capsys, label):
    """T2 on the pixels at least 0.5 px from e1, the degenerate pixel's rule; returns (max error, its distance from e1)."""
    n = len(P1)
    ref, terr, de = geometry(name, P1.tobytes(), P2.tobytes(), n)
    keep = np.broadcast_to(de >= 0.5, ref.shape[:-1])
    far_k, far_r = np.abs(locs).max(-1) >= 50, np.abs(ref).max(-1) >= 50
    bad = np.argwhere((far_k != far_r) & keep)
    assert not bad.size, "%s: far sets differ at (k, n, y, x) %s" % (label, bad[:8].tolist())
    err = np.abs(loc2feat(locs, H, W) - loc2feat(ref, H, W)).max(-1)
    on = keep & ~far_r
    tol = np.maximum(1e-3, np.where(np.isfinite(terr), terr, 0.0))
    over = np.argwhere(on & (err > tol))
    assert not over.size, "%s: %d samples beyond tolerance, first %s err %.3g" % (label, len(over), over[0].tolist(),
                                                                                 err[tuple(over[0])])
    i = np.unravel_index(np.argmax(np.where(on, err, -1)), err.shape)
    worst, dist = float(err[i]), float(de[i[1:]])
    if name in DEGENERATE:
        y, x = DEGENERATE[name]
        for m in range(n):
            s = loc2feat(locs[:, m, y, x], H, W)                              # [K,2] feature px
            if (np.abs(locs[:, m, y, x]).max(-1) >= 50).all():
                continue                                                      # the far sentinel
            assert np.isfinite(s).all(), (label, s)
            _, e2 = epipoles(P1[m], P2[m])
            e2 = img2feat(e2[:2] / e2[2])
            d = s[-1] - s[0]
            off = np.abs(d[0] * (s[:, 1] - e2[1]) - d[1] * (s[:, 0] - e2[0])) / np.hypot(*d)
            assert off.max() < 1e-2, (label, off.max())
            border = lambda p: min(abs(p[0]), abs(p[0] - (W - 1)), abs(p[1]), abs(p[1] - (H - 1)))
            assert border(s[0]) < 1e-3 and border(s[-1]) < 1e-3, (label, s[0], s[-1])
    with capsys.disabled():
        print("\n%-40s T2 max err %.2e px at %.2f px from e1" % (label, worst, dist))
    return worst, dist


def check_t3(f1, f2, P1, P2, locs, out, attn, corr, label, residual=None, z=None):
    """T3: every pixel, against the C oracle on the emitted locations and the fp64 attention's first maximum; a pixel with an
    fp64 score within 3e-5 of 0 (at most 1 in 1000) is left out of the out / attn / corr_pos comparisons, see fp64_attention."""
    n = len(P1)
    o = c_oracle.forward(rig_cfg(K), f1, f2, P1, P2, locs=locs)
    want = o["out"]
    if z is not None:                                                 # folded z + BN, then the fused feature (ZRESIDUAL)
        wf, bf = (t.double().cpu().numpy() for t in z)
        want = np.einsum("oc,nchw->nohw", wf, want.astype(np.float64)) + bf[None, :, None, None] + want
    if residual is not None:
        want = want + residual
    ra, ill = fp64_attention(f1, f2, locs)
    assert ill.mean() <= 1e-3, (label, int(ill.sum()))
    pick = lambda x: x.transpose(0, 2, 3, 1)[~ill]                   # [pixels, channels or samples]
    assert rel_max(pick(out), pick(want)) < TOL, (label, rel_max(pick(out), pick(want)))
    assert rel_max(pick(attn), pick(o["attn"])) < TOL, (label, rel_max(pick(attn), pick(o["attn"])))
    assert np.abs(attn.sum(1) - 1).max() < 1e-5, label
    far = (np.abs(locs).max(-1) >= 50).all(0)                         # [n,H,W]
    a = attn.transpose(0, 2, 3, 1)[far]
    assert np.abs(a - 1.0 / K).max(initial=0) < 1e-7, label
    if z is None:
        rest = np.zeros_like(out) if residual is None else residual
        assert np.array_equal(out.transpose(0, 2, 3, 1)[far], rest.transpose(0, 2, 3, 1)[far]), label
    for m in range(n):
        px = np.flatnonzero(~ill[m].ravel())
        lm = locs[:, m].reshape(K, H * W, 2)[:, px]
        rc = eo.de_normalize(lm[ra[m][:, px].argmax(0), np.arange(px.size)], H, W, True)
        # a near-tie: a relative gap of the fp64 attention below 1e-5, about what the fp32 scores of C = 64 products carry
        check_corr(corr[m].reshape(H * W, 2)[px], rc, ra[m][:, px], lm, H, W, True, near=1e-5)


def run_pair(f1, f2, P1, P2, variant, **kw):
    items32 = variant == "pipe32"
    force_items32(items32)
    try:
        r = epi.epipolar_fusion(f1, f2, dev(P1), dev(P2), K=K, softmax_scale=SCALE, correct_normalize=True, want_locs=True,
                                variant="pipe" if items32 else variant, **kw)
        torch.cuda.synchronize()
    finally:
        force_items32(False)
    out, corr, attn, locs = r
    return out.float().cpu().numpy(), corr.cpu().numpy(), attn.cpu().numpy(), locs.cpu().numpy()


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", RIGS)
def test_pair_form_vs_fp64(name, variant, dt, capsys):
    P1, P2 = pair_rig(name)
    t1, t2, f1, f2 = inputs(len(P1), DTYPES[dt])
    residual = variant == "auto"
    out, corr, attn, locs = run_pair(t1, t2, P1, P2, variant, add_ref_residual=residual)
    label = "%s %s %s" % (name, variant, dt)
    check_t2(name, P1, P2, locs, capsys, label)
    check_t3(f1, f2, P1, P2, locs, out, attn, corr, label, residual=f1 if residual else None)
    if name.startswith("rig90"):                                      # the rays parallel to the source image plane
        col = np.abs(locs[:, 0, :, 32]).max(-1) >= 50
        assert not col[:, 20:45].any() and col[:, :20].all() and col[:, 45:].all()


@pytest.mark.parametrize("name", RIGS)
def test_sample_locs_entry_point(name):
    """epi.sample_locs shares the device geometry with the warp kernel (an FMA contraction may differ by an ulp)."""
    P1, P2 = pair_rig(name)
    t1, t2, _, _ = inputs(len(P1), torch.float32)
    locs = epi.sample_locs(dev(P1), dev(P2), H, W, K, 4.0, 1.0, True).cpu().numpy()
    _, _, _, wl = run_pair(t1, t2, P1, P2, "warp")
    np.testing.assert_allclose(locs, wl, rtol=1e-5, atol=1e-5)


def opposite(v):
    """index j of view v's opposite view v + 2 among its others (u = j + (j >= v))"""
    u = (v + 2) % 4
    return u - (u > v)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("variant", ["pipe", "sector", "tile", "warp", "auto"])
def test_views_form_opposite_pairs(variant, dt, capsys):
    """V = 4, N = 2: each view's opposite view, from the all-others form and from a source table naming it, against fp64
    (T2, T3); a second call through a persistent cache returns the same bits; a bf16 `out` is the fp32 one rounded once."""
    N = 2
    P = ring_opposite(N)
    feats = syn.features(4 * N, C, H, W, "randn", 7).reshape(4, N, C, H, W)
    tf = dev(feats).to(DTYPES[dt])
    f = tf.float().cpu().numpy()
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=True, want_locs=True, variant=variant)
    with torch.no_grad():
        state = epi.FusionState()
        full = [t.cpu() for t in epi.epipolar_fusion_views(tf, dev(P), state=state, **kw)]
        again = [t.cpu() for t in epi.epipolar_fusion_views(tf, dev(P), state=state, **kw)]
        assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(full, again))
        tab = [t.cpu() for t in epi.epipolar_fusion_views(tf, dev(P), sources=[[2], [3], [0], [1]], **kw)]
        half = epi.epipolar_fusion_views(tf, dev(P), out_dtype=torch.bfloat16, **kw)[0].cpu()
    assert torch.equal(half, full[0].to(torch.bfloat16))
    for form, (out, corr, attn, locs), jof in (("views", full, opposite), ("table", tab, lambda v: 0)):
        for v in range(4):
            j, u = jof(v), (v + 2) % 4
            label = "%s %s %s v%d" % (form, variant, dt, v)
            lv = locs[:, v, j].numpy()
            check_t2("ring_opposite", P[v], P[u], lv, capsys, label)
            check_t3(f[v], f[u], P[v], P[u], lv, out[v, j].float().numpy(), attn[v, j].numpy(), corr[v, j].numpy(), label)


def test_benchmark_shape_views_with_z(capsys):
    """The benchmark's workload: V = 4, N = 1, C = 256, 64x64, K = 64, z + ZRESIDUAL; its opposite pairs against fp64."""
    V, N, c = 4, 1, 256
    P = ring_opposite(N)
    feats = syn.features(V * N, c, H, W, "randn", 9).reshape(V, N, c, H, W)
    z = random_z(c, 5)
    with torch.no_grad():
        out, corr, attn, locs = (t.cpu().numpy() for t in epi.epipolar_fusion_views(
            dev(feats), dev(P), K=K, softmax_scale=SCALE, correct_normalize=True, want_locs=True, z_folded=z, z_residual=True))
    for v in range(V):
        j, u = opposite(v), (v + 2) % 4
        label = "bench-shape z v%d" % v
        check_t2("ring_opposite", P[v], P[u], locs[:, v, j], capsys, label)
        check_t3(feats[v], feats[u], P[v], P[u], locs[:, v, j], out[v, j], attn[v, j], corr[v, j], label, z=z)


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("name", RIGS)
def test_backward_with_cameras(name, deterministic):
    """epipolar_fusion_backward deriving its geometry from the cameras gives, within 1e-4, the gradients of the same backward
    on the warp forward's emitted locations, and those of fp64 autograd there.  grad_out is zero at the degenerate pixel, whose
    undefined line may differ between the two derivations."""
    P1, P2 = pair_rig(name)
    n = len(P1)
    t1, t2, f1, f2 = inputs(n, torch.float32, seed=3)
    _, _, attn, locs = run_pair(t1, t2, P1, P2, "warp")
    g = torch.from_numpy(syn.features(n, C, H, W, "randn", 4)).cuda()
    if name in DEGENERATE:
        g[:, :, DEGENERATE[name][0], DEGENERATE[name][1]] = 0
    kw = dict(K=K, softmax_scale=SCALE, correct_normalize=True, deterministic=deterministic)
    a = epipolar_fusion_backward(t1, t2, dev(P1), dev(P2), dev(attn), g, **kw)
    b = epipolar_fusion_backward(t1, t2, None, None, dev(attn), g, sample_locs_in=dev(locs), **kw)
    torch.cuda.synchronize()
    _, e1, e2 = reference_grads(t1, t2, dev(locs), g, None)
    for x, y, e in zip(a, b, (e1, e2)):
        x, y, e = x.cpu().numpy(), y.cpu().numpy(), e.cpu().numpy()
        assert rel_max(x, y) < TOL, (name, rel_max(x, y))
        assert rel_max(x, e) < TOL, (name, rel_max(x, e))
