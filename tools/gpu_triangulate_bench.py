"""Triangulation of the views' joints (KEYPOINT.TRIANGULATION = 'pymvg'), V = 4 views, J = 17 joints, N frames, N in {1, 64, 4096}:
  kernel     triangulate_views: one launch for all N·J problems, CUDA events over --steps launches
  host       the reference's shape: copy locs and scores to the host, then the numpy oracle's loop over frames and joints
             (oracle/triangulate_oracle.py, one np.linalg.svd per joint); host clock around the copy and the loop
  torch_svd  a timing arm only, not the selection rule: A [N·J, 2V, 4] built on the GPU with the rows of views scoring <= 0.05
             zeroed, then torch.linalg.svd; CUDA events.  Also records whether it raises under set_sync_debug_mode("error").
The eval tail of one frame (N = 1) at the H36M ResNet-50 shape (C = 256, 64x64 maps, K = 64, [4,1] nearest-camera table):
  tail       standard_views_test(fuse_head=True) (fused forward with the 1x1 head, then the peak finder) + triangulate_views,
             eager and replayed from one CUDA graph; CUDA events over --steps steps
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_triangulate_bench.py [--steps 200] [--warmup 20] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import multiview, synthetic as syn
from oracle import triangulate_oracle as to
from tools.gpu_multisource_bench import card

V, J = 4, 17
NS = (1, 64, 4096)


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


def inputs(N):
    rng = np.random.default_rng(N)
    P = np.stack([syn.ring_cameras(V, 256, jitter=30.0, seed=n) for n in range(N)], 1)            # [V,N,3,4]
    X = np.array([0.0, 0.0, 1000.0]) + rng.uniform(-600, 600, (N, J, 3))
    uv = np.einsum("vnrc,njc->vnjr", P, np.concatenate([X, np.ones((N, J, 1))], -1))
    locs = (uv[..., :2] / uv[..., 2:3] + rng.normal(0, 1.0, (V, N, J, 2))).astype(np.float32)
    scores = rng.uniform(-0.2, 1.0, (V, N, J)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t(locs), t(scores), t(P.astype(np.float32))


def torch_svd(locs, scores, P):
    M = P[:, :, None].expand(V, P.shape[1], J, 3, 4)                                               # [V,N,J,3,4]
    rows = torch.stack([locs[..., 0:1] * M[..., 2, :] - M[..., 0, :], locs[..., 1:2] * M[..., 2, :] - M[..., 1, :]], 3)
    rows = rows * (scores > 0.05)[..., None, None]                                                  # [V,N,J,2,4]
    A = rows.permute(1, 2, 0, 3, 4).reshape(-1, 2 * V, 4).double()
    vh = torch.linalg.svd(A, full_matrices=False)[2]
    return vh[:, -1, :3] / vh[:, -1, 3:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_triangulate_bench needs a GPU")
    name, q = card()
    print("card: %s  power limit, max SM clock: %s" % (name, q))
    rows = []
    for N in NS:
        locs, scores, P = inputs(N)
        row = dict(N=N, problems=N * J)
        row["kernel_ms"] = events(lambda: epi.triangulate_views(locs, scores, P), args.steps, args.warmup)
        reps = max(1, 64 // N)
        Pn = P.cpu().numpy()                                  # the cameras are on the host already in the reference
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            to.triangulate_loop(locs.cpu().numpy(), scores.cpu().numpy(), Pn)
        row["host_ms"] = (time.perf_counter() - t0) * 1e3 / reps
        row["torch_svd_ms"] = events(lambda: torch_svd(locs, scores, P), max(1, args.steps // 10), 3)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            torch_svd(locs, scores, P)
            row["torch_svd_syncs"] = False
        except RuntimeError as e:
            row["torch_svd_syncs"] = str(e).splitlines()[0][:120]
        finally:
            torch.cuda.set_sync_debug_mode("default")
        rows.append(row)
        print(json.dumps(row))
    # ---- the eval tail of one frame ----
    C, H, W, K = 256, 64, 64, 64
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True))
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    head = torch.nn.Conv2d(C, J, 1).cuda().eval().requires_grad_(False)
    KRT = syn.ring_cameras(V, 4 * H, seed=1, jitter=20.0)
    P = torch.from_numpy(KRT[:, None].astype(np.float32)).cuda()
    src = multiview.nearest_view_table(KRT, topk=1)
    feats = torch.from_numpy(syn.features(V, C, H, W, "randn", 2)[:, None].copy()).cuda()

    def tail():
        locs, scores, _, _ = epi.standard_views_test(m, head, feats, P, src, 2.0, 4.0, fuse_head=True)
        return epi.triangulate_views(locs, scores, P)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.no_grad():
        tail()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        tail()
    with torch.no_grad():
        row = dict(tail="standard_views_test(fuse_head) + triangulate_views, N = 1",
                   eager_ms=events(tail, args.steps, args.warmup), graph_ms=events(g.replay, args.steps, args.warmup))
    rows.append(row)
    print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, limits=q, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
