"""The recursive pictorial structure (KEYPOINT.TRIANGULATION = 'rpsm'), V = 4 views, J = 17 joints, 64x64 and 96x96 heat-maps,
N in {1, 64, 1024} frames, the reference's defaults (16^3 bins of 2000 mm, 10 recursions on 2^3 bins, 150 mm tolerance):
  kernel     rpsm_views: 7 launches for all N frames; CUDA events over --steps calls
  loop       the reference's shape on CUDA tensors, one frame at a time: a grid_sample per view and joint, a dense B x B
             pairwise·energy product and torch.max per edge with a copy of the states to the host per tree node, and the ten
             recursions the same way.  Timed on the host clock over min(N, 4) frames and reported per frame and for all N.
The eval tail of one frame (C = 256, 64x64 maps, K = 64): forward_views(head=) then rpsm_views, eager and replayed from one CUDA
graph; CUDA events over --steps steps.  The card's name and power limit are printed with the numbers.  Needs a GPU; writes
nothing unless --json PATH is given.

    python tools/gpu_rpsm_bench.py [--steps 50] [--warmup 5] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch
import torch.nn.functional as F

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from tests.rpsm_scenes import IMG, scene
from tools.gpu_multisource_bench import card

V, J = 4, 17
NS = (1, 64, 1024)
PARENTS = epi.H36M_PARENTS


def events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


# ---- the reference's shape, one frame, on CUDA tensors ----
def cube(size, centre, n):
    g = torch.linspace(-size / 2, size / 2, n, device=centre.device)
    gx, gy, gz = torch.meshgrid(g + centre[0], g + centre[1], g + centre[2], indexing="ij")
    return torch.stack([gx.reshape(-1), gy.reshape(-1), gz.reshape(-1)], 1)


def unaries(heat, grids, P, T, h, w):
    out = [None] * J
    for v in range(V):
        for j in range(J):
            X = grids[0] if len(grids) == 1 else grids[j]
            q = X @ P[v][:, :3].t() + P[v][:, 3]
            xy = q[:, :2] / q[:, 2:]
            xy = torch.mm(T[v], torch.cat([xy, torch.ones_like(xy[:, :1])], 1).t())[:2].t()
            xy = xy * torch.tensor([w, h], device=xy.device, dtype=torch.float32) / torch.tensor(IMG, device=xy.device, dtype=torch.float32)
            g = (xy / torch.tensor([h - 1, w - 1], device=xy.device, dtype=torch.float32) * 2 - 1).view(1, 1, -1, 2)
            s = F.grid_sample(heat[v:v + 1, j:j + 1], g, align_corners=False).view(-1)
            out[j] = s if out[j] is None else out[j] + s
    return out


def depth(j):
    d = 0
    while PARENTS[j] != -1:
        j, d = PARENTS[j], d + 1
    return d


def infer(U, pw):
    E, S = {}, {}
    for p in sorted(range(J), key=lambda j: -depth(j)):                         # children before parents
        u = U[p].clone()
        for c in [c for c in range(J) if PARENTS[c] == p]:
            mv, mi = torch.max(pw[(p, c)] * E[c][None], dim=1)
            u = u * mv
            S[c] = mi.cpu().numpy()                                             # the reference's per-node host copy
        E[p] = u
    bins = {0: int(np.argmax(E[0].cpu().numpy()))}
    queue = [0]
    while queue:
        p = queue.pop(0)
        for c in [c for c in range(J) if PARENTS[c] == p]:
            bins[c] = int(S[c][bins[p]])
            queue.append(c)
    return bins


def loop_frame(heat, P, T, root, limb, pw0, h, w):
    g0 = cube(2000.0, root, 16)
    bins = infer(unaries(heat, [g0], P, T, h, w), pw0)
    pose = torch.stack([g0[bins[j]] for j in range(J)])
    size = 2000.0 / 16
    for _ in range(10):
        grids = [cube(size, pose[j], 2) for j in range(J)]
        U = unaries(heat, grids, P, T, h, w)
        pw = {}
        for c in range(1, J):
            p = PARENTS[c]
            d = torch.cdist(grids[p], grids[c]) + 1e-9
            pw[(p, c)] = ((d - float(limb[c - 1])).abs() < 150.0).float()
        bins = infer(U, pw)
        pose = torch.stack([grids[j][bins[j]] for j in range(J)])
        size /= 2
    return pose


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_rpsm_bench needs a GPU")
    name, q = card()
    print("card: %s  power limit, max SM clock: %s" % (name, q))
    rows = []
    for hw in (64, 96):
        for N in NS:
            s = scene(V, N, 1000 + N, hw, hw, "signed")
            t = {k: torch.from_numpy(np.ascontiguousarray(s[k])).cuda() for k in ("heat", "P", "T", "root", "limb")}
            L = s["limb"].astype(np.float64).mean(0).astype(np.float32)
            pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(L), nbins=16)
            row = dict(V=V, J=J, map=hw, N=N)
            row["kernel_ms"] = events(lambda: epi.rpsm_views(t["heat"], t["P"], t["T"], IMG, t["root"], t["limb"], pw),
                                      args.steps, args.warmup)
            row["kernel_ms_per_frame"] = row["kernel_ms"] / N
            dense = {}
            bits = pw.cpu().numpy().view(np.uint32)
            for c in range(1, J):
                m = np.unpackbits(bits[c - 1].view(np.uint8), axis=-1, bitorder="little")[:, :4096]
                dense[(PARENTS[c], c)] = torch.from_numpy(m.astype(np.float32)).cuda()
            frames = min(N, 4)
            loop_frame(t["heat"][:, 0], t["P"][:, 0], t["T"][:, 0], t["root"][0], t["limb"][0], dense, hw, hw)   # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for n in range(frames):
                loop_frame(t["heat"][:, n], t["P"][:, n], t["T"][:, n], t["root"][n], t["limb"][n], dense, hw, hw)
            torch.cuda.synchronize()
            row["loop_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / frames
            row["loop_ms_all_frames"] = row["loop_ms_per_frame"] * N
            row["speedup"] = row["loop_ms_all_frames"] / row["kernel_ms"]
            rows.append(row)
            print(json.dumps(row))
    # ---- one frame of the eval tail: forward_views(head=) -> rpsm_views ----
    C, H, W, K = 256, 64, 64, 64
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True))
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    head = torch.nn.Conv2d(C, J, 1).cuda().eval().requires_grad_(False)
    s = scene(V, 1, 7, H, W, "signed")
    P = torch.from_numpy(s["P"]).cuda()
    T, root, limb = (torch.from_numpy(s[k]).cuda() for k in ("T", "root", "limb"))
    pw = epi.rpsm_pairwise(limb_length=torch.from_numpy(s["limb"][0]), nbins=16)
    feats = torch.from_numpy(syn.features(V, C, H, W, "randn", 2)[:, None].copy()).cuda()

    def tail():
        heat = m.forward_views(feats, P, head=head)[0][:, 0]
        return epi.rpsm_views(heat, P, T, IMG, root, limb, pw)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.no_grad():
        tail()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        tail()
    with torch.no_grad():
        row = dict(tail="forward_views(head=) + rpsm_views, N = 1, C = 256, 64x64", eager_ms=events(tail, args.steps, args.warmup),
                   graph_ms=events(g.replay, args.steps, args.warmup))
    rows.append(row)
    print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, limits=q, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
