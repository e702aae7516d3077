"""Time of the default and the deterministic backward of the fused attention, in one process.

Shapes: N=4, C=256, K=64 on 64x64 and 96x96 maps (ring cameras, randn features), fp32 and bf16 maps, with OTHER_GRAD both
('other1', 'other2') and values only ('other2').  Each backward call runs from the same forward outputs, with a loss that also
touches the attention (grad_attn given), and returns both gradients.  Per configuration the two paths alternate within every
round, each warmed up first, and the rounds alternate which path goes first.  Reported per configuration (median over rounds):
  default_ms / deterministic_ms   CUDA-event time of one backward call (mean over --steps back-to-back calls)
  ratio                           deterministic_ms / default_ms
The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_bwd_bench.py [--steps 50] [--warmup 5] [--rounds 5] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward

N, C, K = 4, 256, 64
SIZES = (64, 96)
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
OTHER_GRADS = {"both": ("other1", "other2"), "other2": ("other2",)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def setup(S, dtype):
    P1, P2 = syn.pairs_from_ring(N, 4 * S)
    P1 = torch.from_numpy(P1.astype(np.float32)).cuda(); P2 = torch.from_numpy(P2.astype(np.float32)).cuda()
    f1 = torch.from_numpy(syn.features(N, C, S, S, "randn", 1)).cuda().to(dtype)
    f2 = torch.from_numpy(syn.features(N, C, S, S, "randn", 2)).cuda().to(dtype)
    out, _, attn, locs = epi.epipolar_fusion(f1, f2, P1, P2, K=K, correct_normalize=True, want_locs=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    g_out = torch.randn(out.shape, device="cuda", generator=g)
    g_attn = 0.3 * torch.randn(attn.shape, device="cuda", generator=g)
    return f1, f2, P1, P2, attn, locs, g_out, g_attn


def time_ms(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bwd_bench needs a GPU")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    rows = []
    for S in SIZES:
        for dname, dtype in DTYPES.items():
            f1, f2, P1, P2, attn, locs, g_out, g_attn = setup(S, dtype)
            for oname, og in OTHER_GRADS.items():
                kw = dict(K=K, correct_normalize=True, grad_attn=g_attn, sample_locs_in=locs,
                          grad_keys="other1" in og, grad_vals="other2" in og)
                paths = {p: (lambda det=(p == "deterministic"): epipolar_fusion_backward(f1, f2, P1, P2, attn, g_out, deterministic=det, **kw))
                         for p in ("default", "deterministic")}
                for fn in paths.values():
                    time_ms(fn, args.warmup)
                ms = {p: [] for p in paths}
                for r in range(args.rounds):
                    for p in (list(paths) if r % 2 == 0 else list(paths)[::-1]):
                        ms[p].append(time_ms(paths[p], args.steps))
                row = dict(size="%dx%d" % (S, S), dtype=dname, other_grad=oname,
                           default_ms=statistics.median(ms["default"]), deterministic_ms=statistics.median(ms["deterministic"]),
                           default_spread_ms=max(ms["default"]) - min(ms["default"]),
                           deterministic_spread_ms=max(ms["deterministic"]) - min(ms["deterministic"]))
                row["ratio"] = row["deterministic_ms"] / row["default_ms"]
                rows.append(row)
                print("%-6s %-5s %-7s default %.3f ms (spread %.3f)  deterministic %.3f ms (spread %.3f)  ratio %.2f" % (
                    row["size"], dname, oname, row["default_ms"], row["default_spread_ms"], row["deterministic_ms"],
                    row["deterministic_spread_ms"], row["ratio"]))
            del f1, f2, attn, locs, g_out, g_attn
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, power=power, N=N, C=C, K=K, steps=args.steps, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
