"""Forward time of the fused path on float32, bfloat16 and float16 feature maps, in one process.

Workload: the H36M ResNet-50 256x256 shape (N=4, C=256, 64x64 maps, K=64) with the folded z epilogue and ZRESIDUAL, through a
persistent FusionState per dtype (as `Epipolar` runs it in eval mode).  The dtypes alternate within every round, each is warmed
up first, and the rounds rotate which dtype goes first.  Reported per dtype (median over rounds):
  step_ms    CUDA-event time of one forward (mean over --steps back-to-back calls)
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3), median over --steps calls
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_lowp_bench.py [--steps 200] [--warmup 20] [--rounds 5] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, synthetic as syn

N, C, H, W, K = 4, 256, 64, 64, 64
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_lowp_bench needs a GPU")
    lib = _lib.load()
    P1, P2 = syn.pairs_from_ring(N, 4 * H)
    P1 = torch.from_numpy(P1.astype(np.float32)).cuda(); P2 = torch.from_numpy(P2.astype(np.float32)).cuda()
    f1 = torch.from_numpy(syn.features(N, C, H, W, "relu_smooth", 1)).cuda()
    f2 = torch.from_numpy(syn.features(N, C, H, W, "relu_smooth", 2)).cuda()
    prm = syn.z_bn_params(C, 3)
    z = torch.nn.Conv2d(C, C, 1).cuda(); bn = epi.ZeroInitBN(C).cuda().eval()
    z.load_state_dict({"weight": torch.from_numpy(prm["z.weight"]), "bias": torch.from_numpy(prm["z.bias"])})
    bn.load_state_dict({"weight": torch.from_numpy(prm["bn.weight"]), "bias": torch.from_numpy(prm["bn.bias"]),
                        "running_mean": torch.from_numpy(prm["bn.running_mean"]), "running_var": torch.from_numpy(prm["bn.running_var"]),
                        "num_batches_tracked": torch.tensor(0)})
    zf = epi.fold_z_bn(z, bn)
    maps = {k: (f1.to(dt), f2.to(dt)) for k, dt in DTYPES.items()}
    states = {k: epi.FusionState() for k in DTYPES}
    kw = dict(K=K, downsample=4.0, img_scale=1.0, softmax_scale=1.0 / 8.0, correct_normalize=True, z_folded=zf, z_residual=True,
              want_attn=True, want_corr=True)

    def call(k):
        return epi.epipolar_fusion(*maps[k], P1, P2, state=states[k], **kw)

    # results agree with the float32 call on the upcast maps (what the feature promises), checked once at the timed size
    ref = {k: epi.epipolar_fusion(maps[k][0].float(), maps[k][1].float(), P1, P2, **kw) for k in DTYPES}
    for k in DTYPES:
        got = call(k)
        assert all(torch.equal(g, r) for g, r in zip(got, ref[k]) if r is not None), k
    for k in DTYPES:                                   # warm-up of every dtype before any timed window
        for _ in range(args.warmup):
            call(k)
    torch.cuda.synchronize()

    res = {k: {"step_ms": [], "stage_ms": [], "fused_ms": [], "epilogue_ms": []} for k in DTYPES}
    order = list(DTYPES)
    ms3 = (ctypes.c_float * 3)()
    for r in range(args.rounds):
        rot = order[r % len(order):] + order[:r % len(order)]
        for k in rot:
            for _ in range(3):
                call(k)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                call(k)
            e1.record()
            e1.synchronize()
            res[k]["step_ms"].append(e0.elapsed_time(e1) / args.steps)
            lib.epi_kernel_timing_enable(1)
            groups = []
            for _ in range(args.steps):
                call(k)
                _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                groups.append(list(ms3))
            lib.epi_kernel_timing_enable(0)
            for name, v in zip(("stage_ms", "fused_ms", "epilogue_ms"), np.median(np.array(groups), 0)):
                res[k][name].append(float(v))
    name, plimit = card()
    summary = {"card": name, "power_limit,clocks.max.sm": plimit, "shape": dict(N=N, C=C, H=H, W=W, K=K, z=True, zresidual=True),
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "torch": torch.__version__}
    print("card: %s   power limit, max SM clock: %s" % (name, plimit))
    print("%-5s %10s %10s %10s %12s   (ms, median of %d rounds; step = whole forward)" % ("dtype", "step", "stage", "fused", "epilogue", args.rounds))
    for k in DTYPES:
        med = {m: statistics.median(v) for m, v in res[k].items()}
        spread = max(res[k]["step_ms"]) - min(res[k]["step_ms"])
        print("%-5s %10.4f %10.4f %10.4f %12.4f   step spread %.4f" % (k, med["step_ms"], med["stage_ms"], med["fused_ms"], med["epilogue_ms"], spread))
        summary[k] = dict(med, step_spread_ms=spread, rounds=res[k])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
