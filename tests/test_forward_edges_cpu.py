"""CPU anchors of tests/test_gpu_forward_edges.py: the location generators build the cases they claim (full unions of
exactly the kernels' capacities under each kernel's own marking rule, bit-identical tied sims, epipoles at infinity), and
the float64 reference on given locations agrees with the pinned C oracle."""
import numpy as np
import pytest

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from oracle import c_oracle, epipolar_oracle as eo
from tests.util import (check_corr, edge_locs, fp64_reference, full_union_locs, rel_max, stereo_rig, wide_map_locs,
                        with_ties)

SCALE = float(epi.make_cfg().EPIPOLAR.SOFTMAXSCALE)


def grid2pix32(g, size):
    """the kernels' unnormalize (align_corners=False) bit for bit: fp32 g + 1, one fused multiply-add, an exact halving."""
    g1 = (np.asarray(g, np.float32) + np.float32(1)).astype(np.float64)
    return ((g1 * size - 1.0).astype(np.float32) * np.float32(0.5)).astype(np.float64)


def footprints(locs, H, W):
    """The pipelined kernel's marking rule: every in-bounds pixel of the 2x2 footprint of floor(ix, iy).
    -> (x0, y0) [K,P] ints and `in` [K,P] (some tap in bounds)."""
    ix, iy = grid2pix32(locs[..., 0], W), grid2pix32(locs[..., 1], H)
    inb = (ix > -1) & (ix < W) & (iy > -1) & (iy < H)
    return np.floor(np.where(inb, ix, 0)).astype(np.int64), np.floor(np.where(inb, iy, 0)).astype(np.int64), inb


def pipe_marks(locs, H, W):
    """-> pixels [K,P,4] marked by the pipelined kernel (-1: none), and the footprint rows' first pixels [K,P,2]."""
    x0, y0, inb = footprints(locs, H, W)
    px = np.full(x0.shape + (4,), -1, np.int64)
    first = np.full(x0.shape + (2,), -1, np.int64)
    for r in (0, 1):
        y = y0 + r
        rok = inb & (y >= 0) & (y < H)
        for c in (0, 1):
            x = x0 + c
            ok = rok & (x >= 0) & (x < W)
            px[..., 2 * r + c] = np.where(ok, y * W + x, -1)
        first[..., r] = np.where(rok, y * W + np.maximum(x0, 0), -1)
    return px, first


def tile_marks(locs, H, W):
    """The tile kernel's marking rule: the taps with non-zero weight."""
    ix, iy = grid2pix32(locs[..., 0], W), grid2pix32(locs[..., 1], H)
    fx, fy = np.floor(ix), np.floor(iy)
    ax, ay = ix - fx, iy - fy
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    px = np.full(x0.shape + (4,), -1, np.int64)
    for t, (dx, dy, w) in enumerate(((0, 0, (1 - ax) * (1 - ay)), (1, 0, ax * (1 - ay)), (0, 1, (1 - ax) * ay), (1, 1, ax * ay))):
        x, y = x0 + dx, y0 + dy
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H) & (w != 0)
        px[..., t] = np.where(ok, y * W + x, -1)
    return px


def n_unique(marks):
    """distinct non-negative values per row of [P, M] -> [P]"""
    s = np.sort(marks, axis=1)
    new = np.concatenate([np.ones((s.shape[0], 1), bool), s[:, 1:] != s[:, :-1]], 1)
    return (new & (s >= 0)).sum(1)


def per_pixel(marks):
    """[K,P,M] -> [P, K·M]"""
    K, P, M = marks.shape
    return marks.transpose(1, 0, 2).reshape(P, K * M)


def row_words(px, W):
    """(row, 32-pixel word of the row) pair id of pixel ids (-1 stays -1): the row-windowed bitmap's unit"""
    return np.where(px >= 0, (px // W) * 64 + (px % W) // 32, -1)


def test_full_union_pipe_small_map():
    """36x28, K = 64 on the pipelined kernel: every pixel's union is exactly DMAX = 256, two pixels exceed it (so items
    split down to one pixel), and footprint rows straddle 32-bit words of the linear pixel index (the second atomicOr)."""
    H, W, K = 36, 28, 64
    locs = full_union_locs(K, H, W, range(1, 27, 2), range(1, 35, 2), 21)[:, 0].reshape(K, H * W, 2)
    marks, first = pipe_marks(locs, H, W)
    u = per_pixel(marks)
    assert (n_unique(u) == 4 * K).all()
    assert (n_unique(np.concatenate([u[0::2], u[1::2]], 1)) > 256).all()
    straddle = (first >= 0) & (first % 32 == 31)
    assert straddle.sum() > 1000, straddle.sum()


def test_full_union_tile():
    """48x48, K = 120 on the tile kernel (which marks only taps of non-zero weight): 480 = its DMAX per pixel; two exceed it."""
    H, W, K = 48, 48, 120
    locs = full_union_locs(K, H, W, range(0, 47, 2), range(0, 47, 2), 22)[:, 0].reshape(K, H * W, 2)
    u = per_pixel(tile_marks(locs, H, W))
    assert (n_unique(u) == 480).all()
    assert (n_unique(np.concatenate([u[0::2], u[1::2]], 1)) > 480).all()


def test_full_union_pipe_row_windowed():
    """130x136 (above 16384 pixels), K = 64: in the upper half every pixel touches exactly WIN_WORDS = 256 (row, word) pairs
    holding 256 union pixels, and two pixels exceed both; in the lower half the two alternating sets fill exactly 256 pixels
    in 256 pairs together, and one footprint row starts in the last compacted word."""
    H, W, K = 130, 136, 64
    locs = wide_map_locs(K, H, W, seed=23)[:, 0].reshape(K, H * W, 2)
    marks, first = pipe_marks(locs, H, W)
    u = per_pixel(marks)
    half = H // 2 * W
    top = u[:half]
    assert (n_unique(top) == 256).all() and (n_unique(row_words(top, W)) == 256).all()
    pair = np.concatenate([top[0::2], top[1::2]], 1)
    assert (n_unique(pair) > 256).all() and (n_unique(row_words(pair, W)) > 256).all()
    low = u[half:]
    assert (n_unique(low) == 4 * K - 2).all()                     # A or B alone
    ab = np.concatenate([low[0:1], low[1:2]], 1)
    assert n_unique(ab)[0] == 256 and n_unique(row_words(ab, W))[0] == 256
    assert all((low[i] == low[i % 2]).all() for i in range(0, 64))
    # compacted word index of each footprint row's first pixel, in the order of the (row, word) pairs of A ∪ B
    words = np.unique(row_words(ab[0][ab[0] >= 0], W))
    f = first[:, half:half + 2].reshape(-1)
    looked_up = np.searchsorted(words, row_words(f[f >= 0], W))
    assert looked_up.max() == 255
    assert (words[254:] == row_words(np.array([128 * W + 135, 129 * W + 135]), W)).all()    # the same column in two rows


@pytest.mark.parametrize("shape", [(2, 64, 12, 20, 16), (2, 64, 20, 28, 64), (1, 12, 12, 20, 200)])
def test_tied_sims_are_bit_identical(shape):
    """Set c: in fp32 the tied samples' sims are bit for bit equal and each pixel's maximum.  Every other sample that reaches
    it is an edge-mix pixel centre that landed on a copy as well (the same sampled vector): a tie of the same kind."""
    N, C, H, W, K = shape
    f1, f2 = syn.features(N, C, H, W, "randn", 5), syn.features(N, C, H, W, "randn", 6)
    f1[:, :, 5] = 0.0
    f1, f2, locs, tied = with_ties(f1, f2, edge_locs(K, N, H, W, 11), 12)
    assert len(tied) == 8 * N
    for n, y, x, ks in tied:
        samp = eo.grid_sample_bilinear(f2[n], locs[:, n, y:y + 1, x:x + 1], dtype=np.float32)[:, :, 0, 0]      # [K,C]
        sim = (samp * f1[n, :, y, x][None]).sum(1, dtype=np.float32)
        assert np.unique(sim[ks].view(np.uint32)).size == 1 and sim[ks[0]] == sim.max()
        for k in np.flatnonzero(sim == sim.max()):
            assert np.array_equal(samp[k], samp[ks[0]])


def cam_inverse(a):
    """epi_common.cuh cam_inverse (cofactors, fp64), row-major 9 -> 9"""
    c00, c01, c02 = a[4] * a[8] - a[5] * a[7], a[5] * a[6] - a[3] * a[8], a[3] * a[7] - a[4] * a[6]
    i = 1.0 / (a[0] * c00 + a[1] * c01 + a[2] * c02)
    return [c00 * i, (a[2] * a[7] - a[1] * a[8]) * i, (a[1] * a[5] - a[2] * a[4]) * i,
            c01 * i, (a[0] * a[8] - a[2] * a[6]) * i, (a[2] * a[3] - a[0] * a[5]) * i,
            c02 * i, (a[1] * a[6] - a[0] * a[7]) * i, (a[0] * a[4] - a[1] * a[3]) * i]


def epipole(P_from, P_to):
    """the pixel-order kernels' fp64 epipole: P_to·[centre of P_from; 1], from the float32 matrices"""
    A = [float(v) for v in np.asarray(P_from, np.float64)[:, :3].reshape(-1)]
    t = np.asarray(P_from, np.float64)[:, 3]
    ai = cam_inverse(A)
    c = [-(ai[3 * r] * t[0] + ai[3 * r + 1] * t[1] + ai[3 * r + 2] * t[2]) for r in range(3)]
    B = np.asarray(P_to, np.float64)
    return np.array([B[r, 0] * c[0] + B[r, 1] * c[1] + B[r, 2] * c[2] + B[r, 3] for r in range(3)])


def at_infinity(e):
    """the order kernels' branch: !(fabs(e[2]) > 1e-9 * (fabs(e[0]) + fabs(e[1]) + 1e-300))"""
    return not (abs(e[2]) > 1e-9 * (abs(e[0]) + abs(e[1]) + 1e-300))


@pytest.mark.parametrize("img", [64, 256])
def test_rig_epipoles(img):
    """Rectified pair: float32 exact, e[2] == 0 for both epipoles (the source camera in the reference view, which the order
    kernels use, and the reference camera in the source view), so the parallel branch runs.  Near-rectified pairs: both
    epipoles finite and more than 1e4 px from the image."""
    P1, P2 = stereo_rig(2, img, 0.0)
    for n in range(2):
        assert np.array_equal(P2[n].astype(np.float64), np.round(P2[n].astype(np.float64)))
        for e in (epipole(P2[n], P1[n]), epipole(P1[n], P2[n])):
            assert e[2] == 0.0 and at_infinity(e)
    for yaw in (1e-3, 1e-2):
        P1, P2 = stereo_rig(2, img, yaw)
        for n in range(2):
            for e in (epipole(P2[n], P1[n]), epipole(P1[n], P2[n])):
                assert not at_infinity(e)
                assert np.hypot(e[0] / e[2] - img / 2, e[1] / e[2] - img / 2) > 1e4


def test_rectified_reference_geometry_is_all_far():
    """The reference geometry (fp64, both the reference's pinv path and the infinite homography) gives no epipolar line for
    an exactly rectified pair: every pixel on the far sentinel; a near-rectified pair keeps most pixels."""
    H = W = 16
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=8), EPIPOLAR=dict(SAMPLESIZE=8, USE_CORRECT_NORMALIZE=True))
    P1, P2 = stereo_rig(2, 4 * W, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        for geometry in ("reference", "hinf"):
            g = eo.sample_locs(cfg, P1, P2, H, W, 8, np.float64, geometry)
            assert (np.abs(g).max(-1) >= 50).all()
    P1, P2 = stereo_rig(2, 4 * W, 1e-3)
    g = eo.sample_locs(cfg, P1, P2, H, W, 8, np.float64)
    far = (np.abs(g).max(-1) >= 50).all(0)
    assert 0 < far.mean() < 0.5


def oracle_cfg(C, H, W, K, correct):
    return epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=correct))


def compare_with_c_oracle(f1, f2, locs, correct, P=None):
    K, N, H, W, _ = locs.shape
    cfg = oracle_cfg(f1.shape[1], H, W, K, correct)
    P1, P2 = P if P is not None else (np.zeros((N, 3, 4)), np.zeros((N, 3, 4)))
    o = c_oracle.forward(cfg, f1, f2, P1, P2, locs=locs)
    ro, ra, rc = fp64_reference(f1, f2, locs, SCALE, correct)
    assert rel_max(o["out"].reshape(ro.shape), ro) < 1e-5
    assert rel_max(o["attn"].reshape(ra.shape), ra) < 1e-5
    got = o["corr_pos"].reshape(rc.shape)
    for n in range(N):
        assert check_corr(got[n], rc[n], ra[n], locs[:, n].reshape(K, H * W, 2), H, W, correct) <= 2


@pytest.mark.parametrize("locset", ["edges", "ties"])
@pytest.mark.parametrize("correct", [False, True])
def test_fp64_reference_vs_c_oracle_edges(locset, correct):
    """Sets a and c."""
    N, C, H, W, K = 2, 64, 20, 28, 64
    f1, f2 = syn.features(N, C, H, W, "randn", 5), syn.features(N, C, H, W, "randn", 6)
    f1[:, :, 5] = 0.0
    locs = edge_locs(K, N, H, W, 11)
    if locset == "ties":
        f1, f2, locs, _ = with_ties(f1, f2, locs, 12)
    compare_with_c_oracle(f1, f2, locs, correct)


def test_fp64_reference_vs_c_oracle_full_union():
    """Set b (the 36x28 pipelined-kernel case)."""
    N, C, H, W, K = 1, 64, 36, 28, 64
    f1, f2 = syn.features(N, C, H, W, "randn", 31), syn.features(N, C, H, W, "randn", 32)
    compare_with_c_oracle(f1, f2, full_union_locs(K, H, W, range(1, 27, 2), range(1, 35, 2), 21), False)


@pytest.mark.parametrize("yaw", [1e-3, 1e-2])
def test_fp64_reference_vs_c_oracle_near_rectified(yaw):
    """Rig f: the C oracle's own geometry, then the fp64 reference on the locations it emitted."""
    N, C, H, W, K = 2, 32, 16, 16, 16
    P1, P2 = stereo_rig(N, 4 * W, yaw)
    f1, f2 = syn.features(N, C, H, W, "randn", 41), syn.features(N, C, H, W, "randn", 42)
    o = c_oracle.forward(oracle_cfg(C, H, W, K, True), f1, f2, P1, P2)
    compare_with_c_oracle(f1, f2, o["sample_locs"], True, (P1, P2))
