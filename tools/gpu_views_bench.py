"""Forward time of a whole multi-view frame: every one of V = 4 views fused with its three other views, as one
`epipolar_fusion_views` call against V `epipolar_fusion_multi` calls (one per reference view, S = V - 1 sources each), in one
process.

Workload: the H36M ResNet-50 256x256 shape (C=256, 64x64 maps, K=64) with the folded z epilogue and ZRESIDUAL, eval mode, for
N = 1 and N = 4 items per view, in float32 and bfloat16.  The views form has one persistent FusionState; each of the V
multi-source calls has its own (as `Epipolar.forward_multi` per reference view keeps them), so both forms run with warm camera
caches.  The two forms alternate within every round and the rounds rotate which goes first.  Reported per (N, dtype, form),
median over rounds:
  step_ms    CUDA-event time of one frame (all V·(V−1) pairs), mean over --steps back-to-back steps
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3), summed over the calls of a step,
             median over --steps steps
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_views_bench.py [--steps 100] [--warmup 10] [--rounds 5] [--json out.json]
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
from epipolar_transformers_b200 import _lib, synthetic as syn
from tools.gpu_multisource_bench import card

V, C, H, W, K = 4, 256, 64, 64, 64
NS = (1, 4)
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
FORMS = ("views", "4x multi")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_views_bench needs a GPU")
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
    data, views_state, multi_states = {}, {}, {}
    for n in NS:
        # view v of item i is camera v·N + i of a ring of V·N cameras
        P = torch.from_numpy(syn.ring_cameras(V * n, 4 * H).reshape(V, n, 3, 4).astype(np.float32)).cuda()
        f = torch.from_numpy(syn.features(V * n, C, H, W, "relu_smooth", 1).reshape(V, n, C, H, W)).cuda()
        others = [[u for u in range(V) if u != v] for v in range(V)]
        for k, dt in DTYPES.items():
            fk = f.to(dt)
            # per reference view v: its other views' maps and cameras, stacked once outside the timed loop
            data[(n, k)] = (fk, P, [(fk[v], fk[o].contiguous(), P[v], P[o].contiguous()) for v, o in enumerate(others)])
            views_state[(n, k)] = epi.FusionState()
            multi_states[(n, k)] = [epi.FusionState() for _ in range(V)]

    def views(c):
        fk, P, _ = data[c]
        return [epi.epipolar_fusion_views(fk, P, state=views_state[c], **kw)]

    def multis(c):
        return [epi.epipolar_fusion_multi(a, b, pa, pb, state=multi_states[c][v], **kw) for v, (a, b, pa, pb) in enumerate(data[c][2])]

    calls = {"views": views, "4x multi": multis}
    with torch.no_grad():
        for c in cases:                                  # the two forms agree bit for bit (what the feature promises)
            a, m = views(c)[0], multis(c)
            for i in range(3):
                assert torch.equal(a[i], torch.stack([x[i] for x in m])), (c, i)
        for c in cases:
            for f in FORMS:
                for _ in range(args.warmup):
                    calls[f](c)
        torch.cuda.synchronize()

        res = {(c, f): {"step_ms": [], "stage_ms": [], "fused_ms": [], "epilogue_ms": []} for c in cases for f in FORMS}
        ms3 = (ctypes.c_float * 3)()
        for r in range(args.rounds):
            for c in cases:
                order = FORMS if r % 2 == 0 else FORMS[::-1]
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
                        acc = np.zeros(3)
                        if f == "views":
                            views(c)
                            _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                            acc += np.array(list(ms3))
                        else:
                            for v, (a, b, pa, pb) in enumerate(data[c][2]):
                                epi.epipolar_fusion_multi(a, b, pa, pb, state=multi_states[c][v], **kw)
                                _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                                acc += np.array(list(ms3))
                        groups.append(acc)
                    lib.epi_kernel_timing_enable(0)
                    for name, v in zip(("stage_ms", "fused_ms", "epilogue_ms"), np.median(np.array(groups), 0)):
                        res[(c, f)][name].append(float(v))
    name, plimit = card()
    summary = {"card": name, "power_limit,clocks.max.sm": plimit,
               "shape": dict(V=V, N=list(NS), C=C, H=H, W=W, K=K, z=True, zresidual=True),
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "torch": torch.__version__}
    print("card: %s   power limit, max SM clock: %s" % (name, plimit))
    print("%-3s %-5s %-9s %10s %10s %10s %12s   (ms per frame of V = %d views, %d pairs per item; median of %d rounds)" %
          ("N", "dtype", "form", "step", "stage", "fused", "epilogue", V, V * (V - 1), args.rounds))
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
