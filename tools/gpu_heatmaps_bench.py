"""Eval step of the pose network from the fusion layer to the heat-maps, in two arms, in one process:
  heat      one heat-map call: the 1x1 head (J = 17) as the fused forward's epilogue, z / BN and the head folded once
  unfused   the fused forward (folded z epilogue) + the caller's `ret + feat` + `final_layer` (nn.Conv2d, PyTorch)
Workloads (the H36M ResNet-50 256x256 shape: C=256, 64x64 maps, K=64, z with ZRESIDUAL, float32, eval):
  cfg2      the pair form, N = 4
  t41_n1    the views form with the [4,1] nearest-camera table, N = 1 item per view
  t41_n4    the same, N = 4
The arms alternate within every round and the rounds rotate which goes first.  Reported per (workload, arm), median over rounds:
  step_ms   CUDA-event time of one step, mean over --steps back-to-back steps
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3) of the heat call, median over --steps
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_heatmaps_bench.py [--steps 100] [--warmup 10] [--rounds 5] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, multiview, synthetic as syn
from tools.gpu_multisource_bench import card

C, H, W, K, J = 256, 64, 64, 64, 17
WORKLOADS = {"cfg2": ("pair", 4), "t41_n1": ("table", 1), "t41_n4": ("table", 4)}
ARMS = ("heat", "unfused")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_heatmaps_bench needs a GPU")
    lib = _lib.load()
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                       EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True, PARAMETERIZED=("z",), ZRESIDUAL=True))
    m = epi.Epipolar(cfg=cfg).cuda().eval()
    prm = syn.z_bn_params(C, 3)
    with torch.no_grad():
        m.z.weight.copy_(torch.from_numpy(prm["z.weight"])); m.z.bias.copy_(torch.from_numpy(prm["z.bias"]))
        m.bn.weight.copy_(torch.from_numpy(prm["bn.weight"])); m.bn.bias.copy_(torch.from_numpy(prm["bn.bias"]))
        m.bn.running_mean.copy_(torch.from_numpy(prm["bn.running_mean"]))
        m.bn.running_var.copy_(torch.from_numpy(prm["bn.running_var"]))
    head = torch.nn.Conv2d(C, J, 1).cuda().eval()
    name, q = card()
    print("card: %s  power limit, max SM clock: %s" % (name, q))
    steps = {}
    for wl, (form, N) in WORKLOADS.items():
        V = 4
        KRT = syn.ring_cameras(V * N, 4 * H, seed=1, jitter=20.0).reshape(V, N, 3, 4).astype(np.float32)
        feats = torch.from_numpy(syn.features(V * N, C, H, W, "randn", 2).reshape(V, N, C, H, W)).cuda()
        P = torch.from_numpy(KRT).cuda()
        src = multiview.nearest_view_table(KRT[:, 0], topk=1)
        if form == "pair":
            f1, f2, P1, P2 = feats[0], feats[1], P[0], P[1]
            arms = {"heat": lambda: m.forward_heatmaps(f1, f2, P1, P2, head),
                    "unfused": lambda: head(m(f1, f2, P1, P2)[0] + f1)}
        else:
            arms = {"heat": lambda: m.forward_views(feats, P, sources=src, head=head),
                    "unfused": lambda: head((m.forward_views(feats, P, sources=src)[0] + feats[:, None]).flatten(0, 2))}
        for r in range(args.rounds):
            order = ARMS if r % 2 == 0 else ARMS[::-1]
            for arm in order:
                fn = arms[arm]
                with torch.no_grad():
                    for _ in range(args.warmup):
                        fn()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn()
                    e1.record()
                    torch.cuda.synchronize()
                    groups = []
                    if arm == "heat":
                        lib.epi_kernel_timing_enable(1)
                        ms3 = (ctypes.c_float * 3)()
                        for _ in range(args.steps):
                            fn()
                            lib.epi_kernel_timing_last3(ms3)
                            groups.append(list(ms3))
                        lib.epi_kernel_timing_enable(0)
                steps.setdefault((wl, arm), []).append((e0.elapsed_time(e1) / args.steps,
                                                        [statistics.median(g[i] for g in groups) for i in range(3)] if groups else None))
    res = []
    for (wl, arm), v in steps.items():
        row = dict(workload=wl, arm=arm, step_ms=statistics.median(s for s, _ in v))
        if v[0][1] is not None:
            for i, k in enumerate(("stage_ms", "fused_ms", "epilogue_ms")):
                row[k] = statistics.median(g[i] for _, g in v)
        res.append(row)
        print(json.dumps(row))
    for wl in WORKLOADS:
        h = next(r for r in res if r["workload"] == wl and r["arm"] == "heat")["step_ms"]
        u = next(r for r in res if r["workload"] == wl and r["arm"] == "unfused")["step_ms"]
        print("%s: heat %.4f ms, unfused %.4f ms, saving %.1f %%" % (wl, h, u, 100.0 * (u - h) / u))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, limits=q, rows=res), f, indent=1)


if __name__ == "__main__":
    main()
