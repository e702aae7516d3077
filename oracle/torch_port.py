"""TEST / BASELINE INFRASTRUCTURE — CPU port of the reference's op composition.  NOT product code.

The reference is pure PyTorch (SURVEY.md fact 1) and cannot travel to the GPU box, so the CPU
baseline that bench.py reports ("cpu_baseline", `--impl reference`) is this port: it issues the
SAME ATen operators in the same order and with the same tensor shapes as
/root/reference/modeling/layers/epipolar.py:188-255 — per batch item two F.grid_sample calls on
the K-expanded source view (:199,:210), mul+sum over C (:295), ==0 mask (:298), scale+softmax
(:306-307), argmax+gather (:237-241), mul+sum over K (:243), then conv1x1 + BN + residual
(:249-253) — so its run time is the reference's run time on the same host cores.  It is also
checked against the golden vectors (tests/test_oracle_golden.py), so it doubles as a third oracle.
Sample locations come from oracle/epipolar_oracle.py ('reference' pinv geometry, <1 % of the CPU time) or, with
`geometry=TorchGeometry(...)`, from the reference's own torch operator sequence (what the same-GPU baseline times).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import epipolar_oracle as eo


class TorchGeometry:
    """grid2sample_locs (/root/reference/modeling/layers/epipolar.py:323-418) as the same sequence of torch operators,
    device-agnostic: per-item pinverse in a Python loop (:336), matmul x3 (:338-346), inverse for the camera centre
    (vision/multiview.py:16-21), cross (:350), the four border intersections with sign-preserving denominators (:369-373),
    stack/repeat + slice assignments (:375-386), the half-open validity masks (:388-393), boolean-mask indexing (:402, a
    device->host sync on CUDA), the far sentinel (:403), linear sampling (:405-409), coord2pix + normalize (:411-415).
    Like the reference, the constants are plain CPU tensors built once and moved to the device on EVERY call
    (:338,354-357,369,399,403,409 — they are attributes, not buffers)."""

    def __init__(self, cfg, H, W):
        ds = float(cfg.BACKBONE.DOWNSAMPLE)
        r = float(cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE)
        y = (torch.arange(0, H, dtype=torch.float) * ds + ds / 2.0 - 0.5) * r
        x = (torch.arange(0, W, dtype=torch.float) * ds + ds / 2.0 - 0.5) * r
        gy, gx = torch.meshgrid(y, x, indexing="ij")
        self.grid = torch.stack((gx, gy, torch.ones_like(gx))).view(3, -1)
        self.xmin, self.xmax, self.ymin, self.ymax = x[0], x[-1], y[0], y[-1]
        self.K = int(cfg.EPIPOLAR.SAMPLESIZE)
        self.steps = (torch.arange(self.K, dtype=torch.float64) / (self.K - 1)).float().view(-1, 1, 1, 1)
        self.two_of_four = torch.tensor([True, True, False, False])
        self.far = torch.tensor([self.xmin - 10000, self.ymin - 10000, self.xmin - 10000, self.ymin - 10000]).view(2, 2)
        self.eps = 0.001
        self.ds, self.r, self.H, self.W = ds, r, H, W
        self.correct = bool(cfg.EPIPOLAR.USE_CORRECT_NORMALIZE)

    def __call__(self, P1, P2):
        N, H, W, eps = P1.shape[0], self.H, self.W, self.eps
        P1inv = torch.stack([p.pinverse() for p in P1])
        X = torch.matmul(P1inv, self.grid.to(P1inv))
        x2 = torch.matmul(P2, X)
        x2 = x2 / x2[:, [2], :]
        A_inv = torch.inverse(P1[:, :, :3])
        centre = torch.cat((-torch.matmul(A_inv, P1[:, :, 3:]), torch.ones_like(P1[:, :1, :1])), 1)
        e2 = torch.matmul(P2, centre).view(N, 3, 1)
        e2 = e2 / e2[:, [2], :]
        l2 = torch.cross(e2.expand_as(x2), x2, dim=1).transpose(1, 2)
        xmin, xmax, ymin, ymax = (t.to(l2) for t in (self.xmin, self.xmax, self.ymin, self.ymax))
        EPS = torch.tensor(eps).to(l2)
        sd = lambda v: torch.sign(v) * torch.max(torch.abs(v), EPS)
        by1 = -(xmin * l2[..., 0] + l2[..., 2]) / sd(l2[..., 1])
        by2 = -(xmax * l2[..., 0] + l2[..., 2]) / sd(l2[..., 1])
        bx0 = -(ymin * l2[..., 1] + l2[..., 2]) / sd(l2[..., 0])
        bx3 = -(ymax * l2[..., 1] + l2[..., 2]) / sd(l2[..., 0])
        inter = torch.stack((bx0, by1, by2, bx3), -1).view(N, H * W, 4, 1).repeat(1, 1, 1, 2)
        inter[..., 0, 1] = ymin; inter[..., 1, 0] = xmin; inter[..., 2, 0] = xmax; inter[..., 3, 1] = ymax
        mask = torch.stack(((bx0 >= xmin + eps) & (bx0 < xmax - eps), (by1 > ymin + eps) & (by1 <= ymax - eps),
                            (by2 >= ymin + eps) & (by2 < ymax - eps), (bx3 > xmin + eps) & (bx3 <= xmax - eps)), -1)
        cnt = mask.sum(-1)
        mask[cnt < 2] = 0
        pick = mask.clone()
        pick[cnt < 2] = self.two_of_four.to(pick)
        valid = inter[pick].view(N, H * W, 2, 2)
        valid[cnt < 2] = self.far.to(valid)
        start = valid[..., 0, :]
        vec = (valid[..., 1, :] - start).view(1, N, H * W, 2)
        locs = start.view(1, N, H * W, 2) + vec * self.steps.to(vec)
        locs = locs / self.r
        locs = (locs + 0.5 - self.ds / 2.0) / self.ds                                      # coord2pix
        out = torch.empty_like(locs)
        if self.correct:                                                                   # normalize, multiview.py:25-37
            out[..., 0] = -1.0 + 2.0 * locs[..., 0] / (W - 1)
            out[..., 1] = -1.0 + 2.0 * locs[..., 1] / (H - 1)
        else:
            out[..., 0] = -1.0 + 2.0 * (locs[..., 0] + 0.5) / W
            out[..., 1] = -1.0 + 2.0 * (locs[..., 1] + 0.5) / H
        return out.view(self.K, N, H, W, 2)


def forward(cfg, feat_ref, feat_src, P_ref, P_src, params=None, locs=None, threads=None, geometry=None):
    """feat_*: torch float32 [N,C,H,W] (CPU for the baseline; a CUDA tensor runs the same ATen op sequence on the
    GPU, which is the "reference PyTorch forward on the same GPU" of BASELINE.md B2); P_*: numpy [N,3,4].
    Returns (finalout, corr_pos, attn)."""
    if threads:
        torch.set_num_threads(int(threads))
    N, C, H, W = feat_ref.shape
    K = int(cfg.EPIPOLAR.SAMPLESIZE)
    scale = float(cfg.EPIPOLAR.SOFTMAXSCALE)
    correct = bool(cfg.EPIPOLAR.USE_CORRECT_NORMALIZE)
    with torch.no_grad():
        if locs is None and geometry is not None:           # the reference's own torch geometry, on the tensors' device
            P1 = torch.as_tensor(np.asarray(P_ref, np.float32)).to(feat_ref.device)
            P2 = torch.as_tensor(np.asarray(P_src, np.float32)).to(feat_ref.device)
            locs = geometry(P1, P2)
        if locs is None:
            locs = eo.sample_locs(cfg, np.asarray(P_ref, np.float32), np.asarray(P_src, np.float32), H, W, K,
                                  dtype=np.float32, geometry="reference")
        grid = locs if isinstance(locs, torch.Tensor) else torch.as_tensor(np.asarray(locs), dtype=torch.float32).to(feat_ref.device)   # [K,N,H,W,2]
        src_k = feat_src.unsqueeze(0).expand(K, N, C, H, W)                      # stride-0 view over K
        fused, corr, weights = [], [], []
        for n in range(N):
            g = grid[:, n]
            keys = F.grid_sample(src_k[:, n], g, align_corners=False)            # [K,C,H,W]
            vals = F.grid_sample(src_k[:, n], g, align_corners=False)            # the reference samples twice (fact 3)
            sim = (keys * feat_ref[n].unsqueeze(0).expand(K, -1, -1, -1)).sum(1)
            sim[sim == 0] = -1e10
            sim = F.softmax(sim * scale, 0)
            top = sim.argmax(0)
            pos = torch.gather(g, 0, top.view(1, H, W, 1).expand(-1, -1, -1, 2)).squeeze(0)
            wh = torch.tensor([W, H], dtype=pos.dtype, device=pos.device)
            corr.append((pos + 1) * (wh - 1) / 2.0 if correct else (pos + 1) * wh / 2.0 - 0.5)      # de_normalize, multiview.py:39-57
            fused.append((vals * sim.view(K, 1, H, W)).sum(0))
            weights.append(sim)
        out = torch.stack(fused)
        if "z" in cfg.EPIPOLAR.PARAMETERIZED:
            p = {k: torch.as_tensor(v).to(out.device) for k, v in params.items()}
            y = F.conv2d(out, p["z.weight"], p["z.bias"])
            y = F.batch_norm(y, p["bn.running_mean"], p["bn.running_var"], p["bn.weight"], p["bn.bias"], False, 0.1, 1e-5)
            out = y + out if cfg.EPIPOLAR.ZRESIDUAL else y
        return out, torch.stack(corr), torch.stack(weights)
