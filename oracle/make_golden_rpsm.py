"""TEST INFRASTRUCTURE — freeze tests/golden/rpsm.npz from the UNMODIFIED reference rpsm() (modeling/pictorial_cuda.py) on CPU.

The reference module imports data.transforms.image, whose real module pulls in torchvision; a stand-in module provides the
two functions rpsm() uses: get_affine_transform (rot = 0) as `crop_affine`, and affine_transform_pts_cuda as the same torch.mm.
The reference's `infer` is wrapped (not changed) to record each level's chosen bins.  Each case is one frame:
  ring / look-at rigs with non-trivial crops, a non-square map, signed (noisy, offset) heat-maps, and both level-0 pairwise
  terms: the limb-length mask the reference's PAIRWISE_FILE holds, and a random general 0/1 mask (rpsm_oracle.golden_mask;
  stored as its seed, since the 32 MB of bits are regenerated exactly).
Stored per case: the inputs, the reference's pose and per-level picks [D+1, J], and each pick's top-two margin under the
oracle's energies (the relative gap between the best and the second-best entry of the max it came from).

    python oracle/make_golden_rpsm.py        # needs the reference tree; writes tests/golden/rpsm.npz
"""
from __future__ import annotations

import importlib
import os
import sys
import types
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.rpsm import H36M_PARENTS, crop_affine, limb_lengths
from oracle import ref_harness as rh
from oracle import rpsm_oracle as ro

OUT = os.path.join(ROOT, "tests", "golden", "rpsm.npz")
J, DEPTH, NR, GRID, TOL = 17, 10, 2, 2000.0, 150.0


def load_reference():
    rh._install_shims()
    warnings.filterwarnings("ignore")
    img = types.ModuleType("data.transforms.image")
    img.get_affine_transform = lambda center, scale, rot, output_size, **kw: crop_affine(center, scale, output_size)

    def affine_transform_pts_cuda(pts, t):
        ph = torch.cat([pts, torch.ones(pts.shape[0], 1, device=pts.device)], dim=1)
        return torch.t(torch.mm(t, torch.t(ph))[:2, :])
    img.affine_transform_pts_cuda = affine_transform_pts_cuda
    for name in ("data", "data.transforms"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules.setdefault(name, m)
    sys.modules["data.transforms.image"] = img
    core = importlib.import_module("core")
    for name, sub in (("modeling", "modeling"), ("modeling.layers", os.path.join("modeling", "layers"))):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(rh.REFERENCE_ROOT, sub)]
        sys.modules.setdefault(name, m)
    return importlib.import_module("modeling.pictorial_cuda"), importlib.import_module("modeling.layers.body"), core.cfg


def lookat_rig(rng, V, target):
    out = np.zeros((V, 3, 4))
    for v in range(V):
        f = rng.uniform(800, 1500)
        K = np.array([[f, 0, rng.uniform(400, 600)], [0, f, rng.uniform(400, 600)], [0, 0, 1]])
        C = rng.standard_normal(3)
        C[2] = abs(C[2]) * 0.3
        C *= rng.uniform(3500, 5500) / np.linalg.norm(C)
        C += target
        z = target + rng.normal(0, 100, 3) - C
        z /= np.linalg.norm(z)
        x = np.cross(z, [0, 0, 1.0])
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        out[v] = K @ np.concatenate([R, -R @ C[:, None]], 1)
    return out


def case(seed, rig, V, h, w, signed, general_mask, img=(256, 256)):
    """one frame: a random 300 mm-limbed pose around a root, its heat-maps in each view's crop, the crop affines"""
    rng = np.random.default_rng(seed)
    X = np.zeros((J, 3))
    X[0] = rng.uniform(-300, 300, 3) + [0, 0, 1000 if rig == "ring" else 0]
    for c in range(1, J):
        d = rng.standard_normal(3)
        X[c] = X[H36M_PARENTS[c]] + rng.uniform(250, 350) * d / np.linalg.norm(d)
    P = syn.ring_cameras(V, 1000, jitter=20.0, seed=seed) if rig == "ring" else lookat_rig(rng, V, X[0])
    uv = np.einsum("vrc,jc->vjr", P, np.concatenate([X, np.ones((J, 1))], 1))
    uv = uv[..., :2] / uv[..., 2:]
    center = uv.mean(1) + rng.normal(0, 20, (V, 2))
    scale = (np.ptp(uv, 1).max(1) * rng.uniform(1.2, 1.5, V) / 200.0)[:, None] * np.array([1.0, 1.0])
    T = crop_affine(center, scale, img)                                           # [V,2,3] float64
    Tf = T.astype(np.float32)
    a = np.einsum("vrc,vjc->vjr", Tf.astype(np.float64), np.concatenate([uv, np.ones((V, J, 1))], -1))   # crop px
    hm = a * np.array([w / img[0], h / img[1]])                                   # heat-map px (x, y)
    ys, xs = np.mgrid[0:h, 0:w]
    sig = 1.0
    heat = np.exp(-((xs - hm[..., 0, None, None]) ** 2 + (ys - hm[..., 1, None, None]) ** 2) / (2 * sig ** 2))
    if signed:
        heat = heat + rng.normal(0, 0.02, heat.shape) - 0.01
    heat = heat.astype(np.float16).astype(np.float32)                            # stored as float16, exactly
    L = limb_lengths(X)
    mask_seed = seed if general_mask else -1
    mask = ro.golden_mask(L, mask_seed, 16, GRID, TOL)
    root = X[0] + rng.normal(0, 30, 3)
    return dict(X=X, P=P.astype(np.float32), center=center, scale=scale, T=Tf, heat=heat, root=root, limb=L, mask=mask, img=img,
                h=h, w=w, mask_seed=mask_seed)


def run_reference(pc, body_mod, cfg, c):
    cfg.DATASETS.IMAGE_SIZE = tuple(c["img"])
    cfg.KEYPOINT.HEATMAP_SIZE = (c["w"], c["h"])
    cfg.PICT_STRUCT.GRID_SIZE, cfg.PICT_STRUCT.FIRST_NBINS = GRID, 16
    cfg.PICT_STRUCT.RECUR_NBINS, cfg.PICT_STRUCT.RECUR_DEPTH, cfg.PICT_STRUCT.LIMB_LENGTH_TOLERANCE = NR, DEPTH, TOL
    cfg.KEYPOINT.ROOTIDX = 0
    body = body_mod.HumanBody()
    edges = [(H36M_PARENTS[j], j) for j in range(1, J)]
    pw = {e: torch.from_numpy(c["mask"][i].astype(np.float32)) for i, e in enumerate(edges)}
    ll = body_mod.compute_limb_length(body, c["X"])
    boxes = [dict(center=c["center"][v], scale=c["scale"][v]) for v in range(len(c["P"]))]
    picks = []
    infer = pc.infer

    def recording_infer(unary, pairwise, body):
        out = infer(unary, pairwise, body)
        picks.append([int(i) for _, i in sorted(out)])
        return out
    pc.infer = recording_infer
    try:
        pose = pc.rpsm(torch.from_numpy(c["P"]), torch.from_numpy(c["heat"]),
                       dict(body=body, boxes=boxes, center=c["root"], pairwise=pw, limb_length=ll))
    finally:
        pc.infer = infer
    return pose.numpy(), np.array(picks)


def margins(c):
    """per level and joint, the relative top-two gap of the max that chose the joint's bin, under the oracle's energies"""
    args = (c["heat"][:, None], c["P"][:, None], c["T"][:, None], c["img"], c["root"][None].astype(np.float32), c["limb"][None],
            c["mask"])
    kw = dict(grid_size=GRID, recur_nbins=NR, recur_depth=DEPTH, tolerance=TOL)
    pose, levels, _ = ro.rpsm(*args, picks=True, **kw)
    t = ro.tree(H36M_PARENTS)
    sizes = ro.level_sizes(GRID, 16, NR, DEPTH)
    out = np.zeros((DEPTH + 1, J))
    heat, P, T = args[0], args[1], args[2]
    prev = None
    for r in range(DEPTH + 1):
        if r == 0:
            X = ro.grid(ro.linspace32(sizes[0], 16), args[4])[:, None].repeat(J, 1)     # [1,J,B,3]
        else:
            X = ro.grid(ro.linspace32(sizes[r], NR), prev)
        U = ro.unary(heat, P, T, c["img"], X[:, 0] if r == 0 else X, False)

        def mp(p, ch, Ec, X=X, r=r):
            if r == 0:
                pw = c["mask"][t["edge_of"][ch]].astype(np.float32)[None]
            else:
                pw = ro.limb_ok(X[:, p, :, None], X[:, ch, None], c["limb"][None, t["edge_of"][ch], None, None], TOL).astype(np.float32)
            rows = (pw * Ec[:, None, :]).astype(np.float32)
            mp.rows[ch] = rows
            return ro.torch_max(rows)
        mp.rows = {}
        bins, E = ro.infer(U, mp, t)
        assert (bins == levels[r]).all()
        for j in range(J):
            vals = E[0, j] if j == t["root"] else mp.rows[j][0, bins[0, t["parents"][j]]]
            top = np.sort(vals.astype(np.float64))[::-1]
            out[r, j] = (top[0] - top[1]) / max(abs(top[0]), 1e-30)
        prev = np.take_along_axis(X, bins[..., None, None], 2)[:, :, 0]
    return pose[0], levels[:, 0], out


CASES = [(1, "ring", 4, 32, 32, False, False), (2, "ring", 4, 32, 24, True, False), (3, "lookat", 4, 32, 32, True, False),
         (4, "lookat", 3, 24, 32, False, True), (5, "ring", 2, 32, 32, True, True), (6, "lookat", 8, 32, 32, True, False)]


def main():
    pc, body_mod, cfg = load_reference()
    torch.set_num_threads(8)
    out = {}
    for i, spec in enumerate(CASES):
        c = case(*spec)
        ref_pose, ref_picks = run_reference(pc, body_mod, cfg, c)
        pose, picks, marg = margins(c)
        same = np.array_equal(pose, ref_pose)
        print("case %d %s: pose equal %s, picks equal %s, min margin %.3g, max |dpose| %.3g mm"
              % (i, spec, same, np.array_equal(picks, ref_picks), marg.min(), np.abs(pose - ref_pose).max()))
        for k, v in (("heat", c["heat"].astype(np.float16)), ("P", c["P"]), ("T", c["T"]), ("root", c["root"]), ("limb", c["limb"]),
                     ("mask_seed", np.array(c["mask_seed"])), ("img", np.array(c["img"])), ("ref_pose", ref_pose), ("ref_picks", ref_picks),
                     ("margin", marg), ("center", c["center"]), ("scale", c["scale"])):
            out["c%d_%s" % (i, k)] = v
    out["n_cases"] = np.array(len(CASES))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
