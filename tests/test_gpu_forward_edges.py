"""GPU: the forward kernels against a float64 restatement (oracle.epipolar_oracle's grid_sample_bilinear / fuse_item in fp64,
first-maximum arg-max) on hand-built sample locations that no epipolar line produces:

  a  edge mix: random points, exact pixel centres, border values, points just beyond the border (partial footprints),
     far points, an all-far pixel column and an all-zero query row
  b  full unions: every sample at the middle of a 2x2 block, so a single pixel's union of taps is exactly the kernel's
     capacity (pipelined kernel: 256 rows, and 256 compacted (row, word) pairs above 16384 pixels; tile kernel: 480 rows)
  c  exact ties at distinct locations: the first maximum must win (torch.argmax, DESIGN a6)
  d  NaN, ±inf and ±1e30 locations: they sample nothing, their sims are masked
and on camera rigs whose epipoles lie at infinity (an exactly rectified pair) or far away (a near-rectified pair).

Pass criteria: out and attn within 1e-4 of max|ref|, attention rows sum to 1 within 1e-5, corr_pos equal to the reference's
(tests/util.py::check_corr: exact ties go to the first index; another index only at a near-tie of the fp64 attention)."""
import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from oracle import c_oracle, epipolar_oracle as eo
from tests.util import (check_corr, corr_close, edge_locs, fp64_reference, full_union_locs, px_err, rel_max, stereo_rig,
                        wide_map_locs, with_nonfinite, with_ties)

pytestmark = pytest.mark.gpu
TOL = 1e-4
SCALE = float(epi.make_cfg().EPIPOLAR.SOFTMAXSCALE)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(f1, f2, locs, variant, correct, align_corners=False):
    K = locs.shape[0]
    out, corr, attn, _ = epi.epipolar_fusion(dev(f1), dev(f2), None, None, K=K, softmax_scale=SCALE, correct_normalize=correct,
                                             align_corners=align_corners, sample_locs_in=dev(locs), variant=variant)
    torch.cuda.synchronize()
    return out.cpu().numpy(), attn.cpu().numpy(), corr.cpu().numpy()


def check(f1, f2, locs, variant, correct, capsys, label, align_corners=False, pixels=None):
    """kernel vs fp64 reference on all pixels, or on `pixels` [N,P] (linear indices) of each item."""
    K, N, H, W, _ = locs.shape
    C = f1.shape[1]
    out, attn, corr = run(f1, f2, locs, variant, correct, align_corners)
    ro, ra, rc = fp64_reference(f1, f2, locs, SCALE, correct, align_corners, pixels)
    if pixels is None:
        pixels = np.broadcast_to(np.arange(H * W), (N, H * W))
    n_idx = np.arange(N)[:, None]
    out = out.reshape(N, C, H * W)[n_idx, :, pixels].transpose(0, 2, 1)
    attn = attn.reshape(N, K, H * W)[n_idx, :, pixels].transpose(0, 2, 1)
    corr = corr.reshape(N, H * W, 2)[n_idx, pixels]
    assert rel_max(out, ro) < TOL, rel_max(out, ro)
    assert rel_max(attn, ra) < TOL, rel_max(attn, ra)
    assert np.abs(attn.sum(1) - 1).max() < 1e-5
    near = 0
    for n in range(N):
        ys, xs = np.divmod(pixels[n], W)
        near += check_corr(corr[n], rc[n], ra[n], locs[:, n, ys, xs], H, W, correct)
    with capsys.disabled():
        print("\n%-44s %-4s correct=%d: out %.2e attn %.2e, near-ties %d" % (label, variant, correct, rel_max(out, ro),
                                                                               rel_max(attn, ra), near))


# ---------------------------------------------------------------------------------------------------------------------
# sets a, c, d
# (N, C, H, W, K) -> variants.  Sides are 4·odd so that pixel centres with dyadic coordinates exist (edge_locs).  The
# pipelined kernel takes injected locations up to K = 64 (4K taps <= its 256-row union), the tile kernel up to 4K <= 480.
EDGE_SHAPES = [
    ((2, 64, 12, 20, 16), ("pipe", "tile", "warp", "auto")),
    ((2, 64, 20, 28, 64), ("pipe", "tile", "warp")),
    ((1, 40, 12, 36, 48), ("pipe", "tile", "warp")),
    ((1, 24, 12, 20, 120), ("tile", "auto")),
    ((1, 12, 12, 20, 200), ("warp",)),
]
EDGE_PARAMS = [pytest.param(shape, v, id="%s-%s" % ("x".join(map(str, shape)), v)) for shape, vs in EDGE_SHAPES for v in vs]


def edge_inputs(shape, locset, seed=11):
    N, C, H, W, K = shape
    f1, f2 = syn.features(N, C, H, W, "randn", 5), syn.features(N, C, H, W, "randn", 6)
    f1[:, :, 5] = 0.0                                        # zero query row: every sample masked, uniform attention
    locs = edge_locs(K, N, H, W, seed)
    if locset == "ties":
        f1, f2, locs, _ = with_ties(f1, f2, locs, seed + 1)
    elif locset == "nonfinite":
        locs = with_nonfinite(locs, seed + 2)
    return f1, f2, locs


@pytest.mark.parametrize("correct", [False, True])
@pytest.mark.parametrize("locset", ["edges", "ties", "nonfinite"])
@pytest.mark.parametrize("shape,variant", EDGE_PARAMS)
def test_edge_locations_vs_fp64(shape, variant, locset, correct, capsys):
    f1, f2, locs = edge_inputs(shape, locset)
    check(f1, f2, locs, variant, correct, capsys, "%s %s" % (locset, shape))


@pytest.mark.parametrize("variant", ["pipe", "tile", "warp"])
@pytest.mark.parametrize("locset", ["edges", "nonfinite"])
def test_edge_locations_align_corners(variant, locset, capsys):
    """align_corners=True unnormalises with (size - 1): the dyadic values stay exact, pixel centres move."""
    f1, f2, locs = edge_inputs((2, 64, 12, 20, 16), locset)
    check(f1, f2, locs, variant, False, capsys, "%s align_corners" % locset, align_corners=True)


def test_ties_go_to_the_first_sample():
    """Set c on every kernel: the tied pixels' correspondence is the location of the first sample of the fp64 attention's
    maximum (a tied copy, or an edge-mix pixel centre that landed on a copy earlier), and pixels whose samples all tie (all
    far, zero query) report sample 0."""
    shape = (2, 64, 20, 28, 64)
    N, C, H, W, K = shape
    f1, f2, locs = edge_inputs(shape, "edges")
    f1, f2, locs, tied = with_ties(f1, f2, locs, 12)
    _, ra, _ = fp64_reference(f1, f2, locs, SCALE, True)
    for variant in ("pipe", "tile", "warp"):
        _, attn, corr = run(f1, f2, locs, variant, True)
        for n, y, x, ks in tied:
            a, r = attn[n, :, y, x], ra[n, :, y * W + x]
            assert a[ks].min() == a.max() and (a[ks] == a[ks[0]]).all(), (variant, a[ks], a.max())
            first = int(np.flatnonzero(r == r.max())[0])
            assert first <= ks[0] and (r[ks] == r.max()).all()
            want = eo.de_normalize(locs[first, n, y, x], H, W, True)
            assert corr_close(corr[n, y, x], want), (variant, n, y, x, ks, first)
        for sl in ((slice(None), 5, slice(None)), (slice(None), slice(None), 3)):       # zero query row, all-far column
            want = eo.de_normalize(locs[0][sl], H, W, True)
            assert corr_close(corr[sl], want).all(), variant
            assert (attn.transpose(0, 2, 3, 1)[sl] == attn.transpose(0, 2, 3, 1)[sl][..., :1]).all()


# ---------------------------------------------------------------------------------------------------------------------
# set b: full unions
FULL_UNION = {
    # odd x0 and y0: disjoint blocks, some footprint rows straddle a 32-bit word of the linear pixel index
    "pipe_36x28": ((1, 64, 36, 28, 64), lambda: full_union_locs(64, 36, 28, range(1, 27, 2), range(1, 35, 2), 21), None),
    "tile_48x48": ((1, 32, 48, 48, 120), lambda: full_union_locs(120, 48, 48, range(0, 47, 2), range(0, 47, 2), 22), 768),
    "pipe_130x136": ((1, 16, 130, 136, 64), lambda: wide_map_locs(seed=23), 1024),
}
FULL_PARAMS = [pytest.param(c, v, id="%s-%s" % (c, v)) for c in FULL_UNION for v in (c.split("_")[0], "auto")]


@pytest.mark.parametrize("case,variant", FULL_PARAMS)
def test_full_unions_vs_fp64(case, variant, capsys):
    """Every work item splits down to single pixels whose union is exactly the kernel's capacity (and, on the 130x136 map,
    half of the rows form unsplit items of 256 rows in 256 compacted words).  Large maps are compared on a random subset of
    the reference pixels (the whole source map is sampled)."""
    (N, C, H, W, K), make, n_px = FULL_UNION[case]
    f1, f2 = syn.features(N, C, H, W, "randn", 31), syn.features(N, C, H, W, "randn", 32)
    locs = make()
    pixels = None
    if n_px:
        rng = np.random.default_rng(5)
        half = H // 2 * W
        pixels = np.sort(np.concatenate([rng.choice(half, n_px // 2, replace=False),
                                         half + rng.choice(H * W - half, n_px // 2, replace=False)]))[None]
    check(f1, f2, locs, variant, False, capsys, case, pixels=pixels)


# ---------------------------------------------------------------------------------------------------------------------
# sets e, f: camera rigs with the epipole at or near infinity
RIG_SHAPES = [(2, 32, 16, 16, 16), (2, 64, 64, 64, 32)]
RIG_VARIANTS = ["pipe", "tile", "sector", "warp", "auto"]


def rig_inputs(shape, yaw):
    N, C, H, W, K = shape
    P1, P2 = stereo_rig(N, 4 * W, yaw)
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True))
    return cfg, syn.features(N, C, H, W, "randn", 41), syn.features(N, C, H, W, "randn", 42), P1, P2


def run_rig(shape, yaw, variant, add_ref_residual=False):
    cfg, f1, f2, P1, P2 = rig_inputs(shape, yaw)
    K = shape[4]
    out, corr, attn, locs = epi.epipolar_fusion(dev(f1), dev(f2), dev(P1), dev(P2), K=K, softmax_scale=SCALE, correct_normalize=True,
                                                add_ref_residual=add_ref_residual, want_locs=True, variant=variant)
    torch.cuda.synchronize()
    return (cfg, f1, f2, P1, P2), [t.cpu().numpy() for t in (out, corr, attn, locs)]


@pytest.mark.parametrize("variant", RIG_VARIANTS)
@pytest.mark.parametrize("shape", RIG_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_rectified_pair_has_no_epipolar_line(shape, variant):
    """R = I, baseline along x: the epipole is at infinity (e[2] == 0 exactly).  The reference geometry puts every pixel on the
    far sentinel and so does every kernel (including the parallel-line branch of both pixel-order kernels): uniform
    attention, out = 0 (the reference residual where it is fused), correspondences at the sentinel, as the C oracle gives."""
    residual = variant == "auto"
    (cfg, f1, f2, P1, P2), (out, corr, attn, locs) = run_rig(shape, 0.0, variant, residual)
    N, C, H, W, K = shape
    o = c_oracle.forward(cfg, f1, f2, P1, P2)
    assert (np.abs(o["sample_locs"]).max(-1) >= 50).all()
    err, far_ok = px_err(locs, o["sample_locs"], H, W)
    assert far_ok and (np.abs(locs).max(-1) >= 50).all()
    np.testing.assert_allclose(locs, o["sample_locs"], rtol=1e-6)
    assert np.abs(attn - 1.0 / K).max() < 1e-7 and np.abs(o["attn"] - 1.0 / K).max() < 1e-7
    assert np.array_equal(out, f1 if residual else np.zeros_like(out))
    assert np.abs(o["out"]).max() == 0.0
    assert corr_close(corr, o["corr_pos"]).all()


@pytest.mark.parametrize("variant", RIG_VARIANTS)
@pytest.mark.parametrize("yaw", [1e-3, 1e-2])
@pytest.mark.parametrize("shape", RIG_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_near_rectified_pair(shape, yaw, variant):
    """Yaw 1e-3 / 1e-2 (epipole 4e4 to 1.6e6 px away, finite branch): T3, the C oracle on the kernel's emitted locations; T2, the
    emitted locations against the reference geometry in fp64: the same far set, every sample within 1e-3 feature px of the
    fp64 epipolar line, and along it at least as close to the fp64 samples as the reference's own fp32 geometry is.  (A
    nearly horizontal line that leaves through the top or bottom border meets it at a grazing angle: there an fp32 rounding
    of the line's height moves the clipped end point along the line by up to 1/slope times as much.)"""
    (cfg, f1, f2, P1, P2), (out, corr, attn, locs) = run_rig(shape, yaw, variant)
    N, C, H, W, K = shape
    o = c_oracle.forward(cfg, f1, f2, P1, P2, locs=locs)
    assert rel_max(out, o["out"]) < TOL
    assert rel_max(attn, o["attn"]) < TOL
    assert np.abs(attn.sum(1) - 1).max() < 1e-5
    assert corr_close(corr, o["corr_pos"]).mean() > 0.99
    ref64 = eo.sample_locs(cfg, P1, P2, H, W, K, np.float64)
    err, far_ok = px_err(locs, ref64, H, W)
    ref_err, _ = px_err(eo.sample_locs(cfg, P1, P2, H, W, K, np.float32), ref64, H, W)
    assert far_ok and err <= max(ref_err, 1e-4), (err, ref_err)
    # distance from the fp64 line, in feature px: grid -> image coordinates (USE_CORRECT_NORMALIZE, downsample 4)
    xs, ys = eo.pixel_axes(cfg, H, W)
    lines = eo.epipolar_lines(P1.astype(np.float64), P2.astype(np.float64), xs, ys).reshape(N, H, W, 3)
    img = (np.stack([(locs[..., 0] + 1) * (W - 1) / 2, (locs[..., 1] + 1) * (H - 1) / 2], -1).astype(np.float64) * 4 + 1.5)
    d = np.abs((img * lines[None, ..., :2]).sum(-1) + lines[None, ..., 2]) / np.hypot(lines[..., 0], lines[..., 1])[None] / 4
    valid = np.abs(locs).max(-1) < 50
    assert valid.mean() > 0.5                                                # most pixels do have a line
    assert d[valid].max() < 1e-3, d[valid].max()
