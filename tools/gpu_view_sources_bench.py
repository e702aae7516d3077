"""Forward time of the standard multi-view test (each of V = 4 views fused with its nearest camera, modeling/model.py:240-247) in
three forms, in one process:
  table     one `epipolar_fusion_views(..., sources=[V,1] table)` call on the V views' maps (one backbone pass)
  gather    `feats[src]` gathered into a source batch inside the timed step, then one `epipolar_fusion` call on V·N pairs
  two-maps  one `epipolar_fusion` call on separately held source maps (the reference's two-pass flow without its second
            backbone pass: the source batch already exists)

Workload: V = 4 ring cameras, the nearest-camera table, the H36M ResNet-50 256x256 shape (C=256, 64x64 maps, K=64) with the
folded z epilogue and ZRESIDUAL, eval mode, for N = 1 and N = 4 items per view, in float32 and bfloat16.  Every form keeps its
own FusionState (warm camera caches).  The forms alternate within every round and the rounds rotate which goes first.  Reported
per (N, dtype, form), median over rounds:
  step_ms    CUDA-event time of one frame (all V pairs), mean over --steps back-to-back steps
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3), median over --steps steps (the
             gather's copy is in step_ms only)
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_view_sources_bench.py [--steps 100] [--warmup 10] [--rounds 5] [--json out.json]
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

V, C, H, W, K = 4, 256, 64, 64, 64
NS = (1, 4)
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
FORMS = ("table", "gather", "two-maps")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_view_sources_bench needs a GPU")
    lib = _lib.load()
    prm = syn.z_bn_params(C, 3)
    z = torch.nn.Conv2d(C, C, 1).cuda(); bn = epi.ZeroInitBN(C).cuda().eval()
    z.load_state_dict({"weight": torch.from_numpy(prm["z.weight"]), "bias": torch.from_numpy(prm["z.bias"])})
    bn.load_state_dict({"weight": torch.from_numpy(prm["bn.weight"]), "bias": torch.from_numpy(prm["bn.bias"]),
                        "running_mean": torch.from_numpy(prm["bn.running_mean"]), "running_var": torch.from_numpy(prm["bn.running_var"]),
                        "num_batches_tracked": torch.tensor(0)})
    zf = epi.fold_z_bn(z, bn)
    kw = dict(K=K, downsample=4.0, img_scale=1.0, softmax_scale=1.0 / 8.0, correct_normalize=True, z_folded=zf, z_residual=True,
              want_attn=True, want_corr=True)
    cases = [(n, k) for n in NS for k in DTYPES]
    data, states = {}, {}
    for n in NS:
        # view v of item i is camera v·N + i of a ring of V·N cameras; the table pairs the views by their item-0 cameras
        P = torch.from_numpy(syn.ring_cameras(V * n, 4 * H).reshape(V, n, 3, 4).astype(np.float32)).cuda()
        f = torch.from_numpy(syn.features(V * n, C, H, W, "relu_smooth", 1).reshape(V, n, C, H, W)).cuda()
        src = multiview.nearest_view_table(P[:, 0])                           # [V,1], once per camera rig
        idx = torch.from_numpy(src[:, 0].astype(np.int64)).cuda()
        P1, P2 = P.flatten(0, 1), P[idx].flatten(0, 1).contiguous()          # cameras are rig constants: gathered once
        for k, dt in DTYPES.items():
            fk = f.to(dt)
            data[(n, k)] = dict(f=fk, P=P, src=src, idx=idx, P1=P1, P2=P2, f1=fk.flatten(0, 1), f2=fk[idx].flatten(0, 1).contiguous())
            states[(n, k)] = {form: epi.FusionState() for form in FORMS}

    def table(c):
        d = data[c]
        return epi.epipolar_fusion_views(d["f"], d["P"], sources=d["src"], state=states[c]["table"], **kw)

    def gather(c):
        d = data[c]
        return epi.epipolar_fusion(d["f1"], d["f"][d["idx"]].flatten(0, 1), d["P1"], d["P2"], state=states[c]["gather"], **kw)

    def two_maps(c):
        d = data[c]
        return epi.epipolar_fusion(d["f1"], d["f2"], d["P1"], d["P2"], state=states[c]["two-maps"], **kw)

    calls = {"table": table, "gather": gather, "two-maps": two_maps}
    with torch.no_grad():
        for c in cases:     # each pair of the table call is bit for bit its own single call (what the feature promises)
            d = data[c]
            a, g, t = table(c), gather(c), two_maps(c)
            for v in range(V):
                u = int(d["src"][v, 0])
                one = epi.epipolar_fusion(d["f"][v], d["f"][u], d["P"][v], d["P"][u], **kw)
                assert all(torch.equal(a[i][v, 0], one[i]) for i in range(3)), (c, v)
            assert all(torch.equal(g[i], t[i]) for i in range(3)), c
        for c in cases:
            for f in FORMS:
                for _ in range(args.warmup):
                    calls[f](c)
        torch.cuda.synchronize()

        res = {(c, f): {"step_ms": [], "stage_ms": [], "fused_ms": [], "epilogue_ms": []} for c in cases for f in FORMS}
        ms3 = (ctypes.c_float * 3)()
        for r in range(args.rounds):
            for c in cases:
                order = FORMS[r % 3:] + FORMS[:r % 3]
                for f in order:
                    for _ in range(3):
                        calls[f](c)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        calls[f](c)
                    e1.record()
                    e1.synchronize()
                    res[(c, f)]["step_ms"].append(e0.elapsed_time(e1) / args.steps)
                    lib.epi_kernel_timing_enable(1)
                    groups = []
                    for _ in range(args.steps):
                        calls[f](c)
                        _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                        groups.append(list(ms3))
                    lib.epi_kernel_timing_enable(0)
                    for name, v in zip(("stage_ms", "fused_ms", "epilogue_ms"), np.median(np.array(groups), 0)):
                        res[(c, f)][name].append(float(v))
    name, plimit = card()
    summary = {"card": name, "power_limit,clocks.max.sm": plimit,
               "shape": dict(V=V, S=1, N=list(NS), C=C, H=H, W=W, K=K, z=True, zresidual=True),
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "torch": torch.__version__}
    print("card: %s   power limit, max SM clock: %s" % (name, plimit))
    print("%-3s %-5s %-9s %10s %10s %10s %12s   (ms per frame of V = %d views, each with its nearest camera; median of %d rounds)" %
          ("N", "dtype", "form", "step", "stage", "fused", "epilogue", V, args.rounds))
    for c in cases:
        for f in FORMS:
            v = res[(c, f)]
            med = {m: statistics.median(x) for m, x in v.items()}
            spread = max(v["step_ms"]) - min(v["step_ms"])
            print("%-3d %-5s %-9s %10.4f %10.4f %10.4f %12.4f   step spread %.4f" %
                  (c[0], c[1], f, med["step_ms"], med["stage_ms"], med["fused_ms"], med["epilogue_ms"], spread))
            summary["N%d/%s/%s" % (c[0], c[1], f)] = dict(med, step_spread_ms=spread, rounds=v)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
