"""CPU: the rpsm oracle (oracle/rpsm_oracle.py) against the golden frames frozen from the unmodified reference rpsm()
(tests/golden/rpsm.npz, oracle/make_golden_rpsm.py); its linspace, pairwise_distance and grid ordering against torch; crop_affine
against cv2; the C ABI's and the Python entry points' refusals, checked without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, build
from oracle import rpsm_oracle as ro

EINVAL = -1
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "rpsm.npz")
# DESIGN.md §3.9: a pick whose top-two relative margin exceeds this cannot be changed by the oracle's and the reference's
# different rounding of the projection
MARGIN_BOUND = 1e-3


def golden_cases():
    g = np.load(GOLDEN)
    return [{k[len("c%d_" % i):]: g[k] for k in g.files if k.startswith("c%d_" % i)} for i in range(int(g["n_cases"]))]


@pytest.mark.parametrize("i", range(6))
def test_oracle_reproduces_reference_golden(i):
    """the oracle's pose equals the reference's bit for bit, and so does every pick whose margin clears the bound (in fact
    every pick does)"""
    c = golden_cases()[i]
    mask = ro.golden_mask(c["limb"], int(c["mask_seed"]))
    pose, picks, _ = ro.rpsm(c["heat"].astype(np.float32)[:, None], c["P"][:, None], c["T"][:, None], tuple(c["img"]),
                             c["root"][None].astype(np.float32), c["limb"][None], mask, picks=True)
    assert np.array_equal(pose[0], c["ref_pose"])
    clear = c["margin"] > MARGIN_BOUND
    assert clear[:3].all()                                                     # the coarse levels all clear it
    assert (picks[:, 0][clear] == c["ref_picks"][clear]).all()
    assert (picks[:, 0] == c["ref_picks"]).all()


def test_golden_covers_the_cases():
    cs = golden_cases()
    assert len(cs) == 6
    assert {c["heat"].shape[0] for c in cs} >= {2, 3, 4, 8}
    assert any(c["heat"].shape[-1] != c["heat"].shape[-2] for c in cs)       # a non-square map
    assert any(c["heat"].min() < 0 for c in cs)                               # signed heat-maps
    assert any(int(c["mask_seed"]) >= 0 for c in cs)                           # a random general mask


def test_linspace_matches_torch():
    rng = np.random.default_rng(0)
    for size in [2000.0, 125.0, 62.5, 2000.0 / 16 / 2 ** 9] + list(rng.uniform(1, 5000, 200)):
        for n in (2, 3, 4, 5, 8, 15, 16):
            assert np.array_equal(ro.linspace32(size, n), torch.linspace(-size / 2, size / 2, n).numpy()), (size, n)


def test_pairwise_distance_matches_torch():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((100000, 3)) * rng.choice([1, 100, 1000], (100000, 1))).astype(np.float32)
    y = (x + rng.standard_normal((100000, 3)) * 300).astype(np.float32)
    want = torch.pairwise_distance(torch.from_numpy(x), torch.from_numpy(y)).numpy() + np.float32(1e-9)
    L = rng.uniform(100, 600, 100000).astype(np.float32)
    tol = 150.0
    assert np.array_equal(ro.limb_ok(x, y, L, tol), np.abs(want - L) < np.float32(tol))
    d = (x - y) + np.float32(1e-6)
    n2 = ro.fma32(d[:, 2], d[:, 2], ro.fma32(d[:, 1], d[:, 1], d[:, 0] * d[:, 0]))
    assert np.array_equal(np.sqrt(n2), torch.pairwise_distance(torch.from_numpy(x), torch.from_numpy(y)).numpy())


def test_grid_ordering_matches_meshgrid():
    c = np.array([12.5, -300.25, 1000.0], np.float32)
    g1 = torch.linspace(-1000.0, 1000.0, 16)
    gx, gy, gz = torch.meshgrid(g1 + float(c[0]), g1 + float(c[1]), g1 + float(c[2]), indexing="ij")
    want = torch.stack([gx.reshape(-1), gy.reshape(-1), gz.reshape(-1)], 1).numpy()
    assert np.array_equal(ro.grid(ro.linspace32(2000.0, 16), c[None])[0], want)


def test_fma32_is_one_rounding():
    rng = np.random.default_rng(2)
    a, b = rng.standard_normal((2, 200000)).astype(np.float32)
    c = (rng.standard_normal(200000) * rng.choice([1e-6, 1, 1e6], 200000)).astype(np.float32)
    exact = [float(np.float32(x)) for x in (a.astype(np.float64) * b + c)]            # float64 reference, checked below
    got = ro.fma32(a, b, c)
    from fractions import Fraction
    for i in rng.choice(200000, 2000, replace=False):
        e = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(e))
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - e), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, (a[i], b[i], c[i])
    assert len(exact) == len(got)


def test_crop_affine_matches_cv2():
    """equal in float32 (as the reference's torch.as_tensor(..., dtype=torch.float) reads it), up to the solves' rounding
    noise in the entries that are exactly 0"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for _ in range(200):
        center = rng.uniform(0, 1000, 2)
        scale = rng.uniform(0.5, 5.0, 2)
        size = (int(rng.choice([256, 384])), int(rng.choice([256, 384])))
        s = scale * 200.0
        src = np.zeros((3, 2), np.float32)
        dst = np.zeros((3, 2), np.float32)
        src[0] = center
        src[1] = center + np.array([0, s[0] * -0.5])
        dst[0] = [size[0] * 0.5, size[1] * 0.5]
        dst[1] = np.array([size[0] * 0.5, size[1] * 0.5]) + np.array([0, size[0] * -0.5], np.float32)
        for p in (src, dst):
            d = p[0] - p[1]
            p[2] = p[1] + np.array([-d[1], d[0]], np.float32)
        want = cv2.getAffineTransform(np.float32(src), np.float32(dst)).astype(np.float32)
        got = epi.crop_affine(center, scale, size).astype(np.float32)
        # the rotation-free affine's off-diagonal entries are 0; each solve leaves its own ~1e-17 of rounding there
        big = np.abs(want) > 1e-6
        assert np.array_equal(got[big], want[big]) and np.abs(got[~big] - want[~big]).max(initial=0) < 1e-12


def test_limb_lengths():
    pose = np.random.default_rng(4).standard_normal((5, 17, 3)) * 300
    L = epi.limb_lengths(pose)
    assert L.shape == (5, 16) and L.dtype == np.float32
    assert np.array_equal(L[:, 2], np.linalg.norm(pose[:, 2] - pose[:, 3], axis=-1).astype(np.float32))
    assert torch.equal(epi.limb_lengths(torch.from_numpy(pose)), torch.from_numpy(L))


# ---- the C ABI -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def params(buf, **over):
    a = ctypes.addressof(buf)
    p = _lib.EpiRpsmParams()
    p.heat = p.P = p.crop = p.root = p.limb_length = p.pairwise = p.pose = p.workspace = a
    par = over.pop("parents", list(epi.H36M_PARENTS))
    p.parents = (ctypes.c_int32 * max(len(par), 1))(*par)
    p.V, p.N, p.J, p.h, p.w = 4, 2, 17, 64, 64
    p.first_nbins, p.recur_nbins, p.recur_depth, p.align_corners = 16, 2, 10, 0
    p.image_size[0] = p.image_size[1] = 256.0
    p.grid_size, p.tolerance = 2000.0, 150.0
    p.workspace_bytes = 1 << 40
    for k, v in over.items():
        if k == "image_size":
            p.image_size[0] = v
        else:
            setattr(p, k, v)
    return p


REFUSALS = {
    "null_heat": (dict(heat=None), b"must be non-null"), "null_parents": (dict(parents_null=True), b"must be non-null"),
    "null_workspace": (dict(workspace=None), b"must be non-null"), "null_pairwise": (dict(pairwise=None), b"must be non-null"),
    "V1": (dict(V=1), b"V must be in [2, 64]"), "V65": (dict(V=65), b"V must be in [2, 64]"), "N0": (dict(N=0), b"N >= 1"),
    "J0": (dict(J=0), b"J must be in [1, 32]"), "J33": (dict(J=33), b"J must be in [1, 32]"),
    "two_roots": (dict(parents=[-1, -1, 0]), b"more than one root"), "no_root": (dict(parents=[1, 0, 1]), b"no root"),
    "cycle": (dict(parents=[-1, 2, 1]), b"not a tree"), "parent_range": (dict(parents=[-1, 5, 0]), b"another joint's index"),
    "self_parent": (dict(parents=[-1, 1, 0]), b"another joint's index"),
    "nbins1": (dict(first_nbins=1), b"first_nbins must be in [2, 16]"), "nbins17": (dict(first_nbins=17), b"first_nbins"),
    "rnbins5": (dict(recur_nbins=5), b"recur_nbins must be in [2, 4]"), "rnbins1": (dict(recur_nbins=1), b"recur_nbins"),
    "depth33": (dict(recur_depth=33), b"recur_depth must be in [0, 32]"), "depth_neg": (dict(recur_depth=-1), b"recur_depth"),
    "h1": (dict(h=1), b"h >= 2"), "w1": (dict(w=1), b"h >= 2"),
    "grid_nan": (dict(grid_size=float("nan")), b"grid_size and tolerance"), "grid0": (dict(grid_size=0.0), b"grid_size"),
    "tol_inf": (dict(tolerance=float("inf")), b"grid_size and tolerance"), "tol_neg": (dict(tolerance=-1.0), b"tolerance"),
    "img0": (dict(image_size=0.0), b"image_size"), "heat_misaligned": (dict(heat_off=2), b"4-byte aligned"),
    "ws_misaligned": (dict(ws_off=16), b"256-byte aligned"), "ws_small": (dict(workspace_bytes=1024), b"epi_rpsm_workspace_bytes"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_abi_refusals(lib, case):
    buf = (ctypes.c_double * 1024)()
    over, msg = dict(REFUSALS[case][0]), REFUSALS[case][1]
    heat_off, ws_off, pnull = over.pop("heat_off", 0), over.pop("ws_off", 0), over.pop("parents_null", False)
    if "parents" in over:
        over["J"] = len(over["parents"])
    p = params(buf, **over)
    if heat_off:
        p.heat = ctypes.addressof(buf) + heat_off
    if ws_off:
        p.workspace = (ctypes.addressof(buf) + 255) // 256 * 256 + ws_off
    if pnull:
        p.parents = ctypes.POINTER(ctypes.c_int32)()
    if case not in ("null_workspace", "ws_misaligned"):
        p.workspace = (ctypes.addressof(buf) + 255) // 256 * 256
    rc = lib.epi_rpsm_f32(ctypes.byref(p), None)
    assert rc == EINVAL
    assert msg in lib.epi_last_error(), lib.epi_last_error()


def test_workspace_bytes(lib):
    buf = (ctypes.c_double * 8)()
    p = params(buf)
    B = 4096
    assert lib.epi_rpsm_workspace_bytes(ctypes.byref(p)) == -(-2 * 17 * B * 4 // 256) * 256 + -(-2 * 16 * B * 2 // 256) * 256
    p.first_nbins = 17
    assert lib.epi_rpsm_workspace_bytes(ctypes.byref(p)) == 0


PACK_REFUSALS = {"both": b"exactly one", "neither": b"exactly one", "null_out": b"packed must be non-null",
                 "E32": b"E must be in [0, 31]", "nbins17": b"nbins must be in [2, 16]", "grid_nan": b"grid_size",
                 "tol0": b"tolerance", "misaligned": b"4-byte aligned"}


@pytest.mark.parametrize("case", sorted(PACK_REFUSALS))
def test_pack_refusals(lib, case):
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)
    args = dict(dense=None, limb=a, E=16, nbins=16, grid=2000.0, tol=150.0, out=a)
    if case == "both":
        args["dense"] = a
    elif case == "neither":
        args["limb"] = None
    elif case == "null_out":
        args["out"] = None
    elif case == "E32":
        args["E"] = 32
    elif case == "nbins17":
        args["nbins"] = 17
    elif case == "grid_nan":
        args["grid"] = float("nan")
    elif case == "tol0":
        args["tol"] = 0.0
    elif case == "misaligned":
        args["out"] = a + 2
    rc = lib.epi_rpsm_pairwise_pack(args["dense"], args["limb"], args["E"], args["nbins"], args["grid"], args["tol"], args["out"], None)
    assert rc == EINVAL
    assert PACK_REFUSALS[case] in lib.epi_last_error(), lib.epi_last_error()


# ---- Python --------------------------------------------------------------------------------------------------------------------
def test_python_refusals():
    V, N, J = 4, 2, 17
    heat, P, T = torch.zeros(V, N, J, 8, 8), torch.zeros(V, N, 3, 4), torch.zeros(V, N, 2, 3)
    root, limb = torch.zeros(N, 3), torch.zeros(N, J - 1)
    pw = torch.zeros(J - 1, 512, 16, dtype=torch.int32)
    with pytest.raises(ValueError, match=r"heat must be \[V,N,J,h,w\]"):
        epi.rpsm_views(heat[0], P, T, (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="P must be"):
        epi.rpsm_views(heat, P[..., :3], T, (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="crop must be"):
        epi.rpsm_views(heat, P, T[:, :1], (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="limb_length must be"):
        epi.rpsm_views(heat, P, T, (256, 256), root, limb[:, :3], pw)
    with pytest.raises(ValueError, match="parents names"):
        epi.rpsm_views(heat[:, :, :5], P, T, (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="pairwise must be"):
        epi.rpsm_views(heat, P, T, (256, 256), root, limb, pw.float())
    with pytest.raises(ValueError, match="nbins"):
        epi.rpsm_views(heat, P, T, (256, 256), root, limb, pw[:, :500])
    with pytest.raises(ValueError, match="2 to 64 views"):
        epi.rpsm_views(heat[:1], P[:1], T[:1], (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="floating-point"):
        epi.rpsm_views(heat, P, T, (256, 256), root.int(), limb, pw)
    with pytest.raises(ValueError, match="grid_size"):
        epi.rpsm_views(heat, P, T, (256, 256), root, limb, pw, grid_size=float("nan"))
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        epi.rpsm_views(heat, P, T, (256, 256), root, limb, pw)
    with pytest.raises(ValueError, match="exactly one"):
        epi.rpsm_pairwise()
    with pytest.raises(ValueError, match="nbins"):
        epi.rpsm_pairwise(limb_length=torch.ones(16), nbins=17)


def test_library_without_rpsm(monkeypatch, tmp_path):
    """the rpsm entry points are new symbols: a library without them still loads, and an rpsm call names the missing probe"""
    old = [s for s in _lib.EXPORTS if s not in _lib.RPSM_EXPORTS]
    assert len(old) == len(_lib.EXPORTS) - 4
    src = tmp_path / "old.c"
    src.write_text("".join("int %s(void) { return %d; }\n" % (s, _lib.EPI_ABI_VERSION if s == "epi_version" else 0) for s in old))
    so = tmp_path / "libold.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    _lib.load()
    with pytest.raises(RuntimeError, match="epi_rpsm.*recursive pictorial structure"):
        epi.rpsm_views(torch.zeros(4, 2, 17, 8, 8), torch.zeros(4, 2, 3, 4), torch.zeros(4, 2, 2, 3), (256, 256), torch.zeros(2, 3),
                       torch.zeros(2, 16), torch.zeros(16, 512, 16, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="epi_rpsm"):
        epi.rpsm_pairwise(limb_length=torch.ones(16))
