"""Forward time with a float32 `out` against a bfloat16 `out` (out_dtype=torch.bfloat16, the float32 result rounded once), in
one process, on three workloads of the H100 benchmark shape (C=256, 64x64 maps, K=64, folded z epilogue with ZRESIDUAL, eval
mode, NCHW `out`):
  cfg2      one `epipolar_fusion` call on N = 4 (reference, source) pairs
  table_N1  one `epipolar_fusion_views(..., sources=[V,1] nearest-camera table)` call, V = 4 views, N = 1 item per view
  table_N4  the same with N = 4
each with float32 and with bfloat16 maps.  Every (workload, maps, out) case keeps its own FusionState (warm camera caches).
The two `out` arms alternate within every round and the rounds swap which goes first.  Before timing, the tool checks that the
bf16 `out` is the fp32 `out` rounded, bit for bit.  Reported per case, median over rounds:
  step_ms    CUDA-event time of one call, mean over --steps back-to-back calls
  stage/fused/epilogue_ms   the library's per-launch-group events (epi_kernel_timing_last3), median over --steps calls
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_out_dtype_bench.py [--steps 100] [--warmup 10] [--rounds 6] [--json out.json]
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
WORKLOADS = ("cfg2", "table_N1", "table_N4")
MAPS = {"fp32": torch.float32, "bf16": torch.bfloat16}
OUTS = {"out_fp32": torch.float32, "out_bf16": torch.bfloat16}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_out_dtype_bench needs a GPU")
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

    calls = {}
    for wl in WORKLOADS:
        for mk, mdt in MAPS.items():
            for ok, odt in OUTS.items():
                st = epi.FusionState()
                if wl == "cfg2":
                    P1, P2 = syn.pairs_from_ring(4, 4 * H)
                    P1, P2 = torch.from_numpy(P1.astype(np.float32)).cuda(), torch.from_numpy(P2.astype(np.float32)).cuda()
                    f1 = torch.from_numpy(syn.features(4, C, H, W, "relu_smooth", 1)).cuda().to(mdt)
                    f2 = torch.from_numpy(syn.features(4, C, H, W, "relu_smooth", 2)).cuda().to(mdt)
                    calls[(wl, mk, ok)] = (lambda f1=f1, f2=f2, P1=P1, P2=P2, st=st, odt=odt:
                                           epi.epipolar_fusion(f1, f2, P1, P2, state=st, out_dtype=odt, **kw))
                else:
                    n = int(wl[-1])
                    P = torch.from_numpy(syn.ring_cameras(V * n, 4 * H).reshape(V, n, 3, 4).astype(np.float32)).cuda()
                    f = torch.from_numpy(syn.features(V * n, C, H, W, "relu_smooth", 1).reshape(V, n, C, H, W)).cuda().to(mdt)
                    src = multiview.nearest_view_table(P[:, 0])
                    calls[(wl, mk, ok)] = (lambda f=f, P=P, src=src, st=st, odt=odt:
                                           epi.epipolar_fusion_views(f, P, sources=src, state=st, out_dtype=odt, **kw))
    cases = [(wl, mk) for wl in WORKLOADS for mk in MAPS]
    with torch.no_grad():
        for wl, mk in cases:
            a, b = calls[(wl, mk, "out_fp32")](), calls[(wl, mk, "out_bf16")]()
            assert a[0].dtype == torch.float32 and b[0].dtype == torch.bfloat16
            assert torch.equal(b[0].view(torch.int16), a[0].to(torch.bfloat16).view(torch.int16)), (wl, mk)
            assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), (wl, mk)
        for c in calls.values():
            for _ in range(args.warmup):
                c()
        torch.cuda.synchronize()

        res = {k: {"step_ms": [], "stage_ms": [], "fused_ms": [], "epilogue_ms": []} for k in calls}
        ms3 = (ctypes.c_float * 3)()
        for r in range(args.rounds):
            for wl, mk in cases:
                order = list(OUTS) if r % 2 == 0 else list(OUTS)[::-1]
                for ok in order:
                    f = calls[(wl, mk, ok)]
                    for _ in range(3):
                        f()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        f()
                    e1.record()
                    e1.synchronize()
                    res[(wl, mk, ok)]["step_ms"].append(e0.elapsed_time(e1) / args.steps)
                    lib.epi_kernel_timing_enable(1)
                    groups = []
                    for _ in range(args.steps):
                        f()
                        _lib.check(lib.epi_kernel_timing_last3(ms3), "epi_kernel_timing_last3")
                        groups.append(list(ms3))
                    lib.epi_kernel_timing_enable(0)
                    for name, v in zip(("stage_ms", "fused_ms", "epilogue_ms"), np.median(np.array(groups), 0)):
                        res[(wl, mk, ok)][name].append(float(v))
    name, plimit = card()
    summary = {"card": name, "power_limit,clocks.max.sm": plimit,
               "shape": dict(C=C, H=H, W=W, K=K, z=True, zresidual=True, cfg2_N=4, table_V=V, table_S=1, table_N=[1, 4]),
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "torch": torch.__version__}
    print("card: %s   power limit, max SM clock: %s" % (name, plimit))
    print("%-9s %-5s %-9s %10s %10s %10s %12s   (ms per call; median of %d rounds)" %
          ("workload", "maps", "out", "step", "stage", "fused", "epilogue", args.rounds))
    for wl, mk in cases:
        for ok in OUTS:
            v = res[(wl, mk, ok)]
            med = {m: statistics.median(x) for m, x in v.items()}
            spread = max(v["step_ms"]) - min(v["step_ms"])
            print("%-9s %-5s %-9s %10.4f %10.4f %10.4f %12.4f   step spread %.4f" %
                  (wl, mk, ok, med["step_ms"], med["stage_ms"], med["fused_ms"], med["epilogue_ms"], spread))
            summary["%s/%s/%s" % (wl, mk, ok)] = dict(med, step_spread_ms=spread, rounds=v)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
