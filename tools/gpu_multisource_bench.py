"""Forward time of one reference batch fused against S = 3 source views: one `epipolar_fusion_multi` call (n_src = 3) against
three single-source `epipolar_fusion` calls, in one process.

Workload: the H36M ResNet-50 256x256 shape (N=4, C=256, 64x64 maps, K=64) with the folded z epilogue and ZRESIDUAL, eval mode, in
float32 and bfloat16.  The multi-source form has one persistent FusionState; each of the three single-source calls has its own
(as three `Epipolar` modules, or one module per source, would keep them), so both forms run with warm camera caches.  The two
forms alternate within every round and the rounds rotate which goes first.  Reported per (dtype, form), median over rounds:
  step_ms    CUDA-event time of one multi-view step (all three sources), mean over --steps back-to-back steps
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3), summed over the calls of a step,
             median over --steps steps
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_multisource_bench.py [--steps 200] [--warmup 20] [--rounds 5] [--json out.json]
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

N, C, H, W, K, S = 4, 256, 64, 64, 64, 3
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
FORMS = ("multi", "3x single")


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
        raise SystemExit("gpu_multisource_bench needs a GPU")
    lib = _lib.load()
    KRT = syn.ring_cameras(N + S, 4 * H)                 # reference item n = view n, its source s = view (n + 1 + s) mod (N + S)
    P1 = torch.from_numpy(KRT[:N].astype(np.float32)).cuda()
    P2 = torch.from_numpy(np.stack([KRT[[(n + 1 + s) % (N + S) for n in range(N)]] for s in range(S)]).astype(np.float32)).cuda()
    f1 = torch.from_numpy(syn.features(N, C, H, W, "relu_smooth", 1)).cuda()
    f2 = torch.from_numpy(syn.features(S * N, C, H, W, "relu_smooth", 2).reshape(S, N, C, H, W)).cuda()
    prm = syn.z_bn_params(C, 3)
    z = torch.nn.Conv2d(C, C, 1).cuda(); bn = epi.ZeroInitBN(C).cuda().eval()
    z.load_state_dict({"weight": torch.from_numpy(prm["z.weight"]), "bias": torch.from_numpy(prm["z.bias"])})
    bn.load_state_dict({"weight": torch.from_numpy(prm["bn.weight"]), "bias": torch.from_numpy(prm["bn.bias"]),
                        "running_mean": torch.from_numpy(prm["bn.running_mean"]), "running_var": torch.from_numpy(prm["bn.running_var"]),
                        "num_batches_tracked": torch.tensor(0)})
    zf = epi.fold_z_bn(z, bn)
    kw = dict(K=K, downsample=4.0, img_scale=1.0, softmax_scale=1.0 / 8.0, correct_normalize=True, z_folded=zf, z_residual=True,
              want_attn=True, want_corr=True)
    maps = {k: (f1.to(dt), f2.to(dt)) for k, dt in DTYPES.items()}
    multi_state = {k: epi.FusionState() for k in DTYPES}
    single_states = {k: [epi.FusionState() for _ in range(S)] for k in DTYPES}

    def multi(k):
        return [epi.epipolar_fusion_multi(maps[k][0], maps[k][1], P1, P2, state=multi_state[k], **kw)]

    def singles(k):
        return [epi.epipolar_fusion(maps[k][0], maps[k][1][s], P1, P2[s], state=single_states[k][s], **kw) for s in range(S)]

    calls = {"multi": multi, "3x single": singles}
    with torch.no_grad():
        for k in DTYPES:                                 # the two forms agree bit for bit (what the feature promises)
            m, sg = multi(k)[0], singles(k)
            for i in range(3):
                assert torch.equal(m[i], torch.stack([x[i] for x in sg])), (k, i)
        for k in DTYPES:
            for f in FORMS:
                for _ in range(args.warmup):
                    calls[f](k)
        torch.cuda.synchronize()

        res = {(k, f): {"step_ms": [], "stage_ms": [], "fused_ms": [], "epilogue_ms": []} for k in DTYPES for f in FORMS}
        ms3 = (ctypes.c_float * 3)()
        for r in range(args.rounds):
            for k in DTYPES:
                order = FORMS if r % 2 == 0 else FORMS[::-1]
                for f in order:
                    for _ in range(3):
                        calls[f](k)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        calls[f](k)
                    e1.record()
                    e1.synchronize()
                    res[(k, f)]["step_ms"].append(e0.elapsed_time(e1) / args.steps)
                    lib.epi_kernel_timing_enable(1)
                    groups = []
                    for _ in range(args.steps):
                        acc = np.zeros(3)
                        if f == "multi":
                            multi(k)
                            _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                            acc += np.array(list(ms3))
                        else:
                            for s in range(S):
                                epi.epipolar_fusion(maps[k][0], maps[k][1][s], P1, P2[s], state=single_states[k][s], **kw)
                                _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                                acc += np.array(list(ms3))
                        groups.append(acc)
                    lib.epi_kernel_timing_enable(0)
                    for name, v in zip(("stage_ms", "fused_ms", "epilogue_ms"), np.median(np.array(groups), 0)):
                        res[(k, f)][name].append(float(v))
    name, plimit = card()
    summary = {"card": name, "power_limit,clocks.max.sm": plimit,
               "shape": dict(N=N, S=S, C=C, H=H, W=W, K=K, z=True, zresidual=True),
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "torch": torch.__version__}
    print("card: %s   power limit, max SM clock: %s" % (name, plimit))
    print("%-5s %-10s %10s %10s %10s %12s   (ms per step of %d sources, median of %d rounds)" %
          ("dtype", "form", "step", "stage", "fused", "epilogue", S, args.rounds))
    for k in DTYPES:
        for f in FORMS:
            v = res[(k, f)]
            med = {m: statistics.median(x) for m, x in v.items()}
            spread = max(v["step_ms"]) - min(v["step_ms"])
            print("%-5s %-10s %10.4f %10.4f %10.4f %12.4f   step spread %.4f" %
                  (k, f, med["step_ms"], med["stage_ms"], med["fused_ms"], med["epilogue_ms"], spread))
            summary["%s/%s" % (k, f)] = dict(med, step_spread_ms=spread, rounds=v)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
