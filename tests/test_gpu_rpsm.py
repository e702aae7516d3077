"""GPU: rpsm_views (csrc/epi_rpsm.cu) against the numpy oracle (oracle/rpsm_oracle.py), bit for bit, on > 2000 frames; the MPJPE
proxy scene through forward_views(head=); no host sync; CUDA-graph replay; producers on the current and on a side stream;
poisoned workspace and output; the launch count."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from oracle import mpjpe_proxy, rpsm_oracle as ro
from tests.rpsm_scenes import IMG, J, scene

pytestmark = pytest.mark.gpu
GRID, TOL = 2000.0, 150.0


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(s, pw_dev, depth=10, align=False, grid_size=GRID):
    return epi.rpsm_views(dev(s["heat"]), dev(s["P"]), dev(s["T"]), IMG, dev(s["root"]), dev(s["limb"]), pw_dev,
                          grid_size=grid_size, recur_depth=depth, tolerance=TOL, align_corners=align)


def oracle(s, mask, depth=10, align=False, grid_size=GRID):
    return ro.rpsm(s["heat"], s["P"], s["T"], IMG, s["root"], s["limb"], mask, grid_size=grid_size, recur_depth=depth,
                   tolerance=TOL, align_corners=align)


def mean_limbs(s):
    return s["limb"].astype(np.float64).mean(0).astype(np.float32)


# (V, N, seed, h, w, kind, outside, nbins, align, general mask)
PARITY = [(2, 360, 1, 32, 32, "clean", False, 8, False, False), (3, 300, 2, 32, 32, "noisy", False, 8, False, True),
          (4, 300, 3, 32, 32, "signed", False, 8, True, False), (8, 200, 4, 32, 32, "signed", True, 8, False, True),
          (4, 300, 5, 24, 32, "noisy", True, 8, True, True), (4, 300, 6, 32, 24, "signed", False, 8, False, False),
          (3, 200, 7, 32, 32, "clean", True, 8, False, False), (4, 24, 8, 32, 32, "signed", False, 16, False, False),
          (4, 24, 9, 24, 32, "noisy", True, 16, True, True)]


@pytest.mark.parametrize("spec", PARITY, ids=lambda s: "V%d_N%d_s%d_%dx%d_%s%s_nb%d%s%s" % (
    s[0], s[1], s[2], s[3], s[4], s[5], "_out" if s[6] else "", s[7], "_ac" if s[8] else "", "_gen" if s[9] else ""))
def test_parity_with_oracle(spec):
    """bit-identical poses; both mask forms (limb lengths packed on the device, a dense general mask); the sum over the
    parametrisation is 2008 frames"""
    V, N, seed, h, w, kind, outside, nbins, align, general = spec
    s = scene(V, N, seed, h, w, kind, outside)
    L = mean_limbs(s)
    if general:
        mask = ro.golden_mask(L, seed, nbins, GRID, TOL, density=0.05)
        pw = epi.rpsm_pairwise(mask=torch.from_numpy(mask.astype(np.float32)), nbins=nbins, grid_size=GRID)
    else:
        mask = ro.pairwise_mask(L, nbins, GRID, TOL)
        pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=nbins, grid_size=GRID, tolerance=TOL)
        assert torch.equal(pw, epi.rpsm_pairwise(mask=torch.from_numpy(mask.astype(np.float32)), nbins=nbins, grid_size=GRID))
    want = oracle(s, mask, align=align)
    got = run(s, pw, align=align).cpu().numpy()
    bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any((1, 2)))
    assert len(bad) == 0, "%d of %d frames differ, first %d" % (len(bad), N, bad[0])
    err = np.linalg.norm(got - s["X"], axis=-1).mean()
    print("%s: %d frames bit-identical, MPJPE to the truth %.2f mm" % (spec, N, err))


def test_parity_frames_total():
    assert sum(s[1] for s in PARITY) >= 2000


@pytest.mark.parametrize("what", ["nan", "inf", "-inf", "mixed"])
def test_nonfinite_heatmaps(what):
    """NaN and ±inf in heat-maps follow torch.max: NaN wins, 0·inf is NaN; the pose still equals the oracle's bit for bit"""
    s = scene(4, 24, 20, 32, 32, "signed")
    rng = np.random.default_rng(21)
    vals = {"nan": [np.nan], "inf": [np.inf], "-inf": [-np.inf], "mixed": [np.nan, np.inf, -np.inf]}[what]
    heat = s["heat"]
    for _ in range(60):
        v, n, j, y, x = (rng.integers(0, k) for k in heat.shape)
        heat[v, n, j, max(0, y - 1):y + 1, max(0, x - 1):x + 1] = rng.choice(vals)
    heat[:, 3] = rng.choice(vals)                                               # a whole frame
    L = mean_limbs(s)
    mask = ro.pairwise_mask(L, 8, GRID, TOL)
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=8)
    want = oracle(s, mask)
    got = run(s, pw).cpu().numpy()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_no_recursion_and_one_joint_tree():
    """recur_depth = 0 returns the level-0 bins; a two-joint tree and other parents arrays"""
    s = scene(4, 16, 30)
    L = mean_limbs(s)
    mask = ro.pairwise_mask(L, 8, GRID, TOL)
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=8)
    assert np.array_equal(run(s, pw, depth=0).cpu().numpy(), oracle(s, mask, depth=0))
    parents = (-1, 0)
    s2 = dict(s, heat=s["heat"][:, :, :2].copy(), limb=s["limb"][:, :1].copy())
    m2 = ro.pairwise_mask(L[:1], 8, GRID, TOL)
    pw2 = epi.rpsm_pairwise(limb_length=torch.from_numpy(L[:1]), nbins=8, parents=parents)
    got = epi.rpsm_views(dev(s2["heat"]), dev(s["P"]), dev(s["T"]), IMG, dev(s["root"]), dev(s2["limb"]), pw2, parents=parents,
                         recur_depth=3).cpu().numpy()
    want = ro.rpsm(s2["heat"], s["P"], s["T"], IMG, s["root"], s2["limb"], m2, parents=parents, recur_depth=3)
    assert np.array_equal(got, want)
    # the root elsewhere than joint 0, and children listed out of index order in the tree's shape
    parents = (3, 3, 1, -1, 2)
    s3 = dict(s, heat=s["heat"][:, :, :5].copy(), limb=s["limb"][:, :4].copy())
    m3 = ro.pairwise_mask(L[:4], 8, GRID, TOL)
    pw3 = epi.rpsm_pairwise(limb_length=torch.from_numpy(L[:4]), nbins=8, parents=parents)
    got = epi.rpsm_views(dev(s3["heat"]), dev(s["P"]), dev(s["T"]), IMG, dev(s["root"]), dev(s3["limb"]), pw3, parents=parents,
                         recur_depth=4, recur_nbins=3).cpu().numpy()
    want = ro.rpsm(s3["heat"], s["P"], s["T"], IMG, s["root"], s3["limb"], m3, parents=parents, recur_depth=4, recur_nbins=3)
    assert np.array_equal(got, want)


def proxy_inputs():
    """the MPJPE proxy scene's heat-maps from forward_views(head=) with its 1x1 head, and its inputs in rpsm_views' layout"""
    d = mpjpe_proxy.build(0)
    m = epi.Epipolar(cfg=d["cfg"]).cuda().eval()
    feats = dev(d["feat_ref"])[:, None]
    KRT = dev(d["KRT"].astype(np.float32))
    head = torch.nn.Conv2d(mpjpe_proxy.C, J, 1, bias=False).cuda()
    head.weight.data.copy_(torch.from_numpy(d["head"])[:, :, None, None])
    V = mpjpe_proxy.V
    T = np.broadcast_to(np.array([[1, 0, 0], [0, 1, 0]], np.float32), (V, 1, 2, 3)).copy()          # the identity crop
    img = (mpjpe_proxy.W * 4, mpjpe_proxy.H * 4)
    joints = d["joints"]
    return d, m, feats, KRT, head, T, img, joints


def test_mpjpe_proxy_chain():
    """forward_views(head=) -> rpsm_views on the proxy scene: the MPJPE equals the oracle chain's on the same heat-maps (to
    0.1 mm; the poses are in fact bit-identical)"""
    d, m, feats, KRT, head, T, img, joints = proxy_inputs()
    with torch.no_grad():
        out = m.forward_views(feats, KRT[:, None], head=head)[0]                   # [V,1,J,H,W]
    heat = out[:, 0].contiguous()                                               # [V,N,J,H,W]
    L = epi.limb_lengths(joints, parents=tuple([-1] + [0] * (J - 1)))
    parents = tuple([-1] + [0] * (J - 1))                                       # a star: the proxy's joints are independent
    root = torch.tensor(joints[0], dtype=torch.float32, device="cuda")[None]
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=16, tolerance=1000.0, parents=parents)
    kw = dict(parents=parents, tolerance=1000.0)
    got = epi.rpsm_views(heat, KRT[:, None], dev(T), img, root, torch.from_numpy(L)[None].cuda(), pw, **kw)
    mask = ro.pairwise_mask(L, 16, GRID, 1000.0)
    want = ro.rpsm(heat.cpu().numpy(), d["KRT"][:, None].astype(np.float32), T, img, root.cpu().numpy(), L[None], mask,
                   parents=parents, tolerance=1000.0)
    eg = np.linalg.norm(got[0].cpu().numpy() - joints, axis=-1).mean()
    ew = np.linalg.norm(want[0] - joints, axis=-1).mean()
    print("MPJPE kernel %.6f mm, oracle %.6f mm" % (eg, ew))
    assert abs(eg - ew) <= 0.1
    assert np.array_equal(got.cpu().numpy(), want)


def test_no_host_sync():
    s = scene(4, 64, 40)
    L = mean_limbs(s)
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=16)
    args = [dev(s[k]) for k in ("heat", "P", "T")] + [IMG] + [dev(s[k]) for k in ("root", "limb")] + [pw]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = epi.rpsm_views(*args)
        args[0] = args[0].half()
        b = epi.rpsm_views(*args)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(a).all() and b.shape == (64, J, 3)


def test_launch_count_independent_of_n():
    lib = _lib.load()
    counts = []
    for N in (1, 1024):
        s = scene(4, N, 41)
        pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(mean_limbs(s)), nbins=16)
        run(s, pw)
        counts.append(lib.epi_last_launch_count())
    torch.cuda.synchronize()
    assert counts[0] == counts[1] == 7, counts                                   # unary, 5 tree depths, recursions


def test_cuda_graph_replay():
    """forward_views(head=) -> rpsm_views captured in one graph: replays on new maps equal eager calls bit for bit"""
    d, m, feats, KRT, head, T, img, joints = proxy_inputs()
    parents = tuple([-1] + [0] * (J - 1))
    L = torch.from_numpy(epi.limb_lengths(joints, parents=parents))
    pw = epi.rpsm_pairwise(limb_length=L, nbins=16, tolerance=1000.0, parents=parents)
    root = torch.tensor(joints[0], dtype=torch.float32, device="cuda")[None]
    Ld, Td = L[None].cuda(), dev(T)

    def chain(f):
        with torch.no_grad():
            heat = m.forward_views(f, KRT[:, None], head=head)[0][:, 0]
        return epi.rpsm_views(heat, KRT[:, None], Td, img, root, Ld, pw, parents=parents, tolerance=1000.0)
    maps = [feats.clone()] + [dev(mpjpe_proxy.build(s)["feat_ref"])[:, None] for s in (1, 2)]
    static = maps[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        chain(static)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = chain(static)
    outs = []
    for f in maps[1:] + maps[:1]:
        static.copy_(f)
        g.replay()
        want = chain(f)
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        outs.append(out.clone())
    assert not torch.equal(outs[0], outs[1])


def test_producers_on_current_and_side_stream():
    a, b = scene(4, 128, 50), scene(4, 128, 51, kind="signed")
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(mean_limbs(a)), nbins=16)
    rest = [dev(a[k]) for k in ("P", "T")] + [IMG] + [dev(a[k]) for k in ("root", "limb")] + [pw]
    ha, hb = dev(a["heat"]), dev(b["heat"])
    want = epi.rpsm_views(hb, *rest)
    other = epi.rpsm_views(ha, *rest)
    torch.cuda.synchronize()
    assert not torch.equal(want, other)
    side = torch.cuda.Stream()
    for producer in ("current", "side"):
        x = ha.clone()
        torch.cuda.synchronize()
        if producer == "current":
            torch.cuda._sleep(50_000_000)
            x.copy_(hb)
        else:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(50_000_000)
                x.copy_(hb)
            torch.cuda.current_stream().wait_stream(side)
        got = epi.rpsm_views(x, *rest)
        torch.cuda.synchronize()
        assert torch.equal(got, want), producer


@pytest.mark.parametrize("poison", [float("nan"), 12345.0])
def test_poisoned_workspace_and_output(poison):
    """workspace and pose prefilled with poison through the C ABI: the pose equals rpsm_views' and the oracle's"""
    s = scene(3, 21, 60, 24, 32, "signed")
    L = mean_limbs(s)
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=16)
    ts = [dev(s[k]) for k in ("heat", "P", "T", "root", "limb")]
    lib = _lib.load()
    par = (ctypes.c_int32 * J)(*epi.H36M_PARENTS)
    pose = torch.full((21, J, 3), poison, device="cuda")
    p = _lib.EpiRpsmParams()
    p.heat, p.P, p.crop, p.root, p.limb_length = (t.data_ptr() for t in ts)
    p.pairwise, p.parents, p.pose = pw.data_ptr(), par, pose.data_ptr()
    p.V, p.N, p.J, p.h, p.w = 3, 21, J, 24, 32
    p.first_nbins, p.recur_nbins, p.recur_depth, p.align_corners = 16, 2, 10, 0
    p.image_size[0], p.image_size[1] = IMG
    p.grid_size, p.tolerance = GRID, TOL
    nbytes = lib.epi_rpsm_workspace_bytes(ctypes.byref(p))
    ws = torch.full((nbytes // 4,), poison, device="cuda")
    p.workspace, p.workspace_bytes = ws.data_ptr(), nbytes
    _lib.check(lib.epi_rpsm_f32(ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "epi_rpsm_f32")
    want = run(s, pw)
    torch.cuda.synchronize()
    assert torch.equal(pose, want)
    assert np.array_equal(pose.cpu().numpy(), oracle(s, ro.pairwise_mask(L, 16, GRID, TOL)))
