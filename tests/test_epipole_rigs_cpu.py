"""CPU: the camera rigs whose epipoles lie inside the maps (tests/util.py::pair_rig), and the oracles' geometry on them.

  - where the epipoles lie, the sign of e1's third coordinate, how far e1 is from a pixel centre;
  - rig90: zz == 0 in fp32 on a whole pixel column (rays parallel to the source image plane), and not on its twin;
  - every fixture is well posed: no fp64 line of a pixel away from e1 is clipped within 1e-4 px of a validity threshold, so
    comparing far sets compares geometry, not rounding;
  - both oracles' infinite-homography geometry (the numpy oracle's geometry='hinf', and epi_oracle.c in fp64 and in fp32)
    against the reference's pinv geometry in fp64, including rig90's zz == 0 column;
  - the reference module's own fp32 geometry (oracle/torch_port.TorchGeometry) against fp64, and its raising on the facing
    rig, where a line meets more than two borders in fp32: the kernels and oracles keep the first two intersections there."""
import numpy as np
import pytest
import torch

from oracle import c_oracle, epipolar_oracle as eo, torch_port
from tests.util import PAIR_RIGS, RIG_HW, e1_distance, epipoles, img2feat, loc2feat, pair_rig, ring_opposite, rig_cfg

H = W = RIG_HW
K = 16
RIGS = ["ring_opposite", "ring_opposite_n1"] + PAIR_RIGS
DEGENERATE = {"facing": (32, 32), "behind": (32, 32)}        # pixels whose ray meets the source camera centre


def rig(name):
    if name == "ring_opposite_n1":                              # the benchmark's rig: V = 4, N = 1
        P = ring_opposite(N=1)
        return P.reshape(-1, 3, 4), P[[2, 3, 0, 1]].reshape(-1, 3, 4)
    return pair_rig(name)


def fp64_lines(P1, P2):
    xs, ys = eo.pixel_axes(rig_cfg(K), H, W)
    return eo.epipolar_lines(P1.astype(np.float64), P2.astype(np.float64), xs, ys).reshape(len(P1), H, W, 3), xs, ys


def test_epipoles_inside():
    """e1 (in the reference view) and e2 (in the source view) in feature px, and the sign of e1's third coordinate."""
    inside = lambda e: bool(((e >= 0) & (e <= H - 1)).all())
    for name in RIGS:
        P1, P2 = rig(name)
        for n in range(len(P1)):
            e1, e2 = epipoles(P1[n], P2[n])
            f1, f2 = img2feat(e1[:2] / e1[2]), img2feat(e2[:2] / e2[2])
            if name.startswith("rig90"):
                assert inside(f1) and not inside(f2) and f2[0] < -150, (name, f1, f2)
            else:
                assert inside(f1) and inside(f2), (name, n, f1, f2)
            assert (e1[2] < 0) == name.startswith("behind"), (name, e1)
            assert e2[2] > 0
            d = np.abs(f1 - np.round(f1)).max()
            if name in DEGENERATE:
                assert d == 0 and tuple(np.round(f1[::-1]).astype(int)) == DEGENERATE[name]
            else:
                assert d > 0.1, (name, n, f1)
            if name == "centre":                                   # the middle of the pixel-centre rectangle exactly
                assert (f1 == (W - 1) / 2).all()


def test_rig90_zz_is_zero_on_a_column():
    """M = A2·A1^-1 rounded to fp32 as the kernels hold it: its third row is (−1/256, 0, 129.5/256), so zz = M6·x + M7·y + M8
    is exactly 0 at x = 129.5 (column 32) for every row, in any evaluation order.  The twin's zz there is tiny but not 0."""
    xs, ys = eo.pixel_axes(rig_cfg(K), H, W, np.float32)
    for name, zero in (("rig90", True), ("rig90_twin", False)):
        P1, P2 = (p[0].astype(np.float64) for p in pair_rig(name))
        M = (P2[:, :3] @ np.linalg.inv(P1[:, :3])).astype(np.float32)
        zz32 = M[2, 0] * xs[32] + M[2, 1] * ys + M[2, 2]
        zz64 = M[2, 0].astype(np.float64) * xs[32] + M[2, 1].astype(np.float64) * ys + M[2, 2]
        if zero:
            assert M[2].tolist() == [np.float32(-1 / 256), 0.0, np.float32(129.5 / 256)]
            assert (zz32 == 0).all() and (zz64 == 0).all()
        else:
            assert (zz32 != 0).all() and (zz64 != 0).all() and np.abs(zz64).max() < 1e-4


@pytest.mark.parametrize("name", RIGS)
def test_fixture_well_posed(name):
    """The four border intersections of every fp64 line, of every pixel at least 0.1 px from e1, lie more than 1e-4 image px
    from each validity threshold (xmin + eps, xmax − eps, ymin + eps, ymax − eps)."""
    P1, P2 = rig(name)
    L, xs, ys = fp64_lines(P1, P2)
    l0, l1, l2 = L[..., 0], L[..., 1], L[..., 2]
    e = eo.EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        cands = [(-(ys[0] * l1 + l2) / eo._sd(l0, e), xs), (-(xs[0] * l0 + l2) / eo._sd(l1, e), ys),
                 (-(xs[-1] * l0 + l2) / eo._sd(l1, e), ys), (-(ys[-1] * l1 + l2) / eo._sd(l0, e), xs)]
    keep = e1_distance(P1, P2, H, W) >= 0.1
    for c, ax in cands:
        for t in (ax[0] + e, ax[-1] - e):
            d = np.abs(c - t)[keep]
            assert np.nan_to_num(d, nan=np.inf).min() > 1e-4, (name, t)


@pytest.mark.parametrize("name", RIGS)
def test_oracles_pinned_to_reference_geometry(name):
    """geometry='hinf' (with its homogeneous line where x2 has no finite quotient) equals the reference's pinv geometry within
    1e-9 feature px in fp64, far sets equal, on every pixel at least 0.1 px from e1; epi_oracle.c returns the fp64 locations
    rounded to fp32 (within 2 ulp) from its fp64 geometry, and within 1e-3 px from its fp32 geometry."""
    P1, P2 = rig(name)
    cfg = rig_cfg(K)
    ref = eo.sample_locs(cfg, P1, P2, H, W, K, np.float64, "reference")
    hinf = eo.sample_locs(cfg, P1, P2, H, W, K, np.float64, "hinf")
    keep = np.broadcast_to(e1_distance(P1, P2, H, W) >= 0.1, ref.shape[:-1])
    far_r = np.abs(ref).max(-1) >= 50
    assert ((np.abs(hinf).max(-1) >= 50) == far_r)[keep].all()
    assert np.abs(loc2feat(hinf, H, W) - loc2feat(ref, H, W))[keep & ~far_r].max() < 1e-9
    f = np.zeros((len(P1), 1, H, W), np.float32)
    for fp32, tol in ((False, None), (True, 1e-3)):
        c = c_oracle.forward(cfg, f, f, P1, P2, geom_fp32=fp32)["sample_locs"]
        assert ((np.abs(c).max(-1) >= 50) == far_r)[keep].all(), fp32
        if tol is None:
            np.testing.assert_allclose(c[keep], ref[keep], rtol=2 ** -22, atol=2 ** -23)
        else:
            assert np.abs(loc2feat(c, H, W) - loc2feat(ref, H, W))[keep & ~far_r].max() < tol
    if name.startswith("rig90"):                                    # the zz == 0 column has its lines
        assert not far_r[:, 0, 20:45, 32].any() and far_r[:, 0, :20, 32].all() and far_r[:, 0, 45:, 32].all()


@pytest.mark.parametrize("name", RIGS)
def test_reference_module_geometry(name):
    """TorchGeometry, the reference's fp32 operator sequence (pinv per item): the same far set as fp64 and within 0.5 feature
    px of it (its fp32 pinv is noisy on the ring's opposite pairs) on all but a few pixels per rig, whose lines pass near a
    corner, where its rounding picks other borders or another order of the end points.  On the facing rig a line meets more
    than two borders within eps in fp32 and the reference raises at its two-of-four reshape (epipolar.py:402); the kernels
    and oracles keep the first two intersections there."""
    P1, P2 = rig(name)
    geom = torch_port.TorchGeometry(rig_cfg(K), H, W)
    if name == "facing":
        with pytest.raises(RuntimeError):
            geom(torch.from_numpy(P1), torch.from_numpy(P2))
        return
    tg = geom(torch.from_numpy(P1), torch.from_numpy(P2)).numpy()
    ref = eo.sample_locs(rig_cfg(K), P1, P2, H, W, K, np.float64, "reference")
    far_t, far_r = (np.abs(a).max(-1) >= 50 for a in (tg, ref))
    err = np.where(far_t | far_r, 0.0, np.abs(loc2feat(tg, H, W) - loc2feat(ref, H, W)).max(-1))
    off = ((far_t != far_r) | (err >= 0.5)).any(0)
    assert off.sum() <= 4, np.argwhere(off)
    if name == "rig90":                                             # the zz == 0 column: the reference has its lines too
        assert not far_t[:, 0, 20:45, 32].any()
        assert np.abs(loc2feat(tg, H, W) - loc2feat(ref, H, W))[:, 0, 20:45, 32].max() < 1e-3
