"""Training-step time of the views form's backward against the gathered flow, in one process.

Layer (always): V = 4 views, N = 4 frames, each view fused with its nearest camera (S = 1: 16 pairs, the reference's training
batch), C = 256, K = 64, 64x64 and 96x96 maps, float32 and bfloat16 maps, the default and the deterministic backward.  One step
is the forward and the backward of the Epipolar layer in training mode (z + ZRESIDUAL, PyTorch's conv and BatchNorm) under the
loss Σ out·w:
  views     `Epipolar.forward_views_train(feats, P, sources=table)`: each view map is staged once by the forward and once by the
            backward, and the backward returns one gradient per view item
  gathered  `feats[q]` and `feats[u]` gathered into query and source batches inside the step, `Epipolar.forward` under autograd
            and the backward through the gathers (the one-pair backward plus autograd's index_add)
Step (--backbone, only when torchvision imports): a torchvision ResNet-50 (weights=None) with three 256-channel stride-2 deconvs
to 64x64 stands in for the pose network; a full training step (backbone, fusion, 1x1 head, MSE, backward) of the reference's
two-pass flow (backbone on the 16 source images, then on the 16 views) against the one-pass flow (backbone once on the 16 views,
then `forward_views_train`).
The arms alternate within every round and the rounds rotate which goes first; every shape is warmed before the first round.
Reported per case and arm: ms per step, the median over rounds with the min and max, and torch.cuda.max_memory_allocated of a
round.  The card's name and power limit are printed with the numbers.  Needs a GPU; writes nothing unless --json PATH is given.

    python tools/gpu_views_bwd_bench.py [--steps 20] [--warmup 5] [--rounds 5] [--backbone] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch
import torch.nn.functional as F

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import multiview, synthetic as syn
from tools.gpu_multisource_bench import card

V, N, C, K = 4, 4, 256, 64
SIZES = (64, 96)
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
ARMS = ("views", "gathered")


def make_layer(H, W):
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                       EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True, PARAMETERIZED=("z",), ZRESIDUAL=True))
    m = epi.Epipolar(cfg=cfg).cuda().train()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.z_bn_params(C, 3).items()}, strict=False)
    return m


def rig(H):
    P = torch.from_numpy(syn.ring_cameras(V * N, 4 * H).reshape(V, N, 3, 4).astype(np.float32)).cuda()
    src = multiview.nearest_view_table(P[:, 0])                                   # [V,1]
    q = torch.arange(V * N, device="cuda")
    u = torch.from_numpy(np.repeat(src[:, 0].astype(np.int64) * N, N) + np.tile(np.arange(N), V)).cuda()
    return P, src, q, u


def layer_steps(m, feats, P, src, q, u, w):
    """-> {arm: step()}: one forward + backward of the layer from the V·N view maps"""
    Pf = P.flatten(0, 1)
    Pq, Pu = Pf[q].contiguous(), Pf[u].contiguous()

    def views():
        x = feats.detach().requires_grad_(True)
        out = m.forward_views_train(x, P, sources=src)[0]
        (out.flatten(0, 2) * w).sum().backward()

    def gathered():
        x = feats.detach().requires_grad_(True)
        xf = x.flatten(0, 1)
        out = m(xf.index_select(0, q), xf.index_select(0, u), Pq, Pu)[0]
        (out * w).sum().backward()

    return {"views": views, "gathered": gathered}


def timed(fn, steps):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated() / 2**20


def run_rounds(cases, steps, warmup, rounds):
    """cases: {name: {arm: fn}} -> {name: {arm: (median, min, max, peak MB)}}"""
    for arms in cases.values():
        for fn in arms.values():
            for _ in range(warmup):
                fn()
    res = {name: {arm: [] for arm in arms} for name, arms in cases.items()}
    mem = {name: {arm: 0.0 for arm in arms} for name, arms in cases.items()}
    for r in range(rounds):
        for name, arms in cases.items():
            order = list(arms)
            order = order[r % len(order):] + order[:r % len(order)]
            for arm in order:
                ms, mb = timed(arms[arm], steps)
                res[name][arm].append(ms)
                mem[name][arm] = max(mem[name][arm], mb)
    return {name: {arm: (statistics.median(v), min(v), max(v), mem[name][arm]) for arm, v in arms.items()}
            for name, arms in res.items()}


class PoseNet(torch.nn.Module):
    """torchvision ResNet-50 (no pretrained weights) + three 256-channel stride-2 deconvs: 256x256 images -> 64x64 maps"""

    def __init__(self):
        super().__init__()
        import torchvision
        r = torchvision.models.resnet50(weights=None)
        self.body = torch.nn.Sequential(r.conv1, r.bn1, r.relu, r.maxpool, r.layer1, r.layer2, r.layer3, r.layer4)
        layers, cin = [], 2048
        for _ in range(3):
            layers += [torch.nn.ConvTranspose2d(cin, 256, 4, 2, 1, bias=False), torch.nn.BatchNorm2d(256), torch.nn.ReLU()]
            cin = 256
        self.deconv = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.deconv(self.body(x))


def step_cases(det):
    torch.manual_seed(0)
    H = W = 64
    net = torch.nn.ModuleDict(dict(backbone=PoseNet(), epi=make_layer(H, W), head=torch.nn.Conv2d(C, 17, 1))).cuda().train()
    P, src, q, u = rig(H)
    g = torch.Generator(device="cuda").manual_seed(1)
    img = torch.randn((V * N, 3, 4 * H, 4 * W), device="cuda", generator=g)
    target = torch.randn((V * N, 17, H, W), device="cuda", generator=g)
    Pf = P.flatten(0, 1)
    Pu = Pf[u].contiguous()

    def two_pass():
        net.zero_grad(set_to_none=True)
        other = net["backbone"](img.index_select(0, u))
        feat = net["backbone"](img)
        ret = net["epi"](feat, other, Pf, Pu)[0]
        F.mse_loss(net["head"](ret + feat), target).backward()

    def one_pass():
        net.zero_grad(set_to_none=True)
        feats = net["backbone"](img).unflatten(0, (V, N))
        ret = net["epi"].forward_views_train(feats, P, sources=src)[0]
        F.mse_loss(net["head"](ret[:, 0].flatten(0, 1) + feats.flatten(0, 1)), target).backward()

    return {"step_r50_%s" % ("det" if det else "default"): {"two-pass": two_pass, "one-pass": one_pass}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--backbone", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_views_bwd_bench needs a GPU")
    torch.backends.cudnn.benchmark = False
    name, limits = card()
    print("card: %s | power limit, max SM clock: %s" % (name, limits))
    results = {}
    for det in (False, True):
        torch.use_deterministic_algorithms(det, warn_only=True)
        for H in SIZES:
            m = make_layer(H, H)
            P, src, q, u = rig(H)
            f = torch.from_numpy(syn.features(V * N, C, H, H, "relu_smooth", 1).reshape(V, N, C, H, H)).cuda()
            w = torch.randn((V * N, C, H, H), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
            cases = {"%dx%d_%s_%s" % (H, H, k, "det" if det else "default"): layer_steps(m, f.to(dt), P, src, q, u, w)
                     for k, dt in DTYPES.items()}
            results.update(run_rounds(cases, args.steps, args.warmup, args.rounds))
        if args.backbone:
            try:
                import torchvision  # noqa: F401
            except ImportError:
                print("--backbone: torchvision does not import; step comparison skipped")
            else:
                results.update(run_rounds(step_cases(det), max(1, args.steps // 4), args.warmup, args.rounds))
    torch.use_deterministic_algorithms(False)
    print("%-26s %-10s %10s %10s %10s %10s" % ("case", "arm", "ms/step", "min", "max", "peak MB"))
    for case, arms in results.items():
        for arm, (med, lo, hi, mb) in arms.items():
            print("%-26s %-10s %10.3f %10.3f %10.3f %10.0f" % (case, arm, med, lo, hi, mb))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=name, limits=limits, steps=args.steps, rounds=args.rounds, results=results), fh, indent=1)


if __name__ == "__main__":
    main()
