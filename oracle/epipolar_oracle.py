"""TEST INFRASTRUCTURE — CPU oracle for the epipolar fusion path.  NOT product code.

A numpy restatement of the reference algorithm, each function citing the reference lines
it follows (paths relative to /root/reference).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this package; the product
(epipolar_transformers_b200) never does and fails loudly without its CUDA library.

Pinning: the reference ships NO golden vectors or tests for this path (SURVEY.md section 4),
so this restatement is pinned against outputs of the reference module itself, executed in
the build container by oracle/make_golden.py and committed under tests/golden/
(tests/test_oracle_golden.py).  Third-party arithmetic boundary = PyTorch
(F.grid_sample / softmax / pinverse of the installed torch 2.11, align_corners=False).
"""
from __future__ import annotations

import numpy as np

EPS = 1e-3            # epipolar.py:20   self.epsilon
FAR = 10000.0         # epipolar.py:51-53 outrange sentinel offset
MASKED = -1e10        # epipolar.py:298  sim[sim==0] = -1e10


# ------------------------------------------------------------------------------------------
# constants of Epipolar.__init__                                    (epipolar.py:22-54)
# ------------------------------------------------------------------------------------------
def pixel_axes(cfg, H, W, dtype=np.float64):
    """Image-space coordinates of feature-pixel centres: pix2coord (vision/multiview.py:154-157)
    times IMAGE_RESIZE*PREDICT_RESIZE (epipolar.py:35-38).  The reference builds them in fp32."""
    ds = cfg.BACKBONE.DOWNSAMPLE
    r = cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE
    f32 = np.float32
    ys = (np.arange(H, dtype=f32) * f32(ds) + f32(ds / 2.0) - f32(0.5)) * f32(r)
    xs = (np.arange(W, dtype=f32) * f32(ds) + f32(ds / 2.0) - f32(0.5)) * f32(r)
    return xs.astype(dtype), ys.astype(dtype)


def sample_steps(K, dtype=np.float64):
    """torch.range(0, 1, 1/(K-1)) (epipolar.py:54) == k/(K-1), exactly K points (SURVEY app. B)."""
    return (np.arange(K, dtype=np.float64) / (K - 1)).astype(dtype)


# ------------------------------------------------------------------------------------------
# geometry: grid2sample_locs                                        (epipolar.py:323-418)
# ------------------------------------------------------------------------------------------
def _sd(v, eps):
    """sign(v) * max(|v|, eps)  (epipolar.py:370-373)."""
    return np.sign(v) * np.maximum(np.abs(v), eps)


def epipolar_lines(P_ref, P_src, xs, ys, geometry="reference"):
    """Per-pixel epipolar line l = e2 x x2 in the source image -> [N, H*W, 3].

    geometry='reference': x2 = P2 (pinv(P1) p), e2 = P2 [-A1^-1 t1; 1], both divided by their
      third component (epipolar.py:336-350, vision/multiview.py:16-21).
    geometry='hinf': the better-conditioned point on the SAME line x2' = (A2 A1^-1) p and
      e2 = A2 (-A1^-1 t1) + t2 (SURVEY.md appendix B) — what the CUDA kernel evaluates.  Where x2' has no finite
      quotient (a ray parallel to the source image plane: x2'[2] == 0), the line is e2 × x2' of the homogeneous point, the
      limit of the quotient form up to a factor that grows without bound; it is scaled so that its smallest non-zero
      direction component is 1, so the eps clamp of the clipping denominators does not act on it (as in that limit).
    """
    dt = P_ref.dtype
    N = P_ref.shape[0]
    gx, gy = np.meshgrid(xs, ys)                      # [H,W]; index = y*W+x (epipolar.py:40-44)
    grid = np.stack([gx.ravel(), gy.ravel(), np.ones(gx.size, dtype=dt)]).astype(dt)   # [3,HW]
    lines = np.zeros((N, grid.shape[1], 3), dtype=dt)
    for n in range(N):
        P1, P2 = P_ref[n], P_src[n]
        A1inv = np.linalg.inv(P1[:, :3])
        center = -A1inv @ P1[:, 3]
        if geometry == "reference":
            X = np.linalg.pinv(P1) @ grid                                # [4,HW]
            x2 = P2 @ X
            e2 = P2 @ np.concatenate([center, [1.0]]).astype(dt)
        elif geometry == "hinf":
            x2 = (P2[:, :3] @ A1inv) @ grid
            e2 = P2[:, :3] @ center + P2[:, 3]
        else:
            raise ValueError(geometry)
        e2 = e2 / e2[2]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            l = np.cross(np.broadcast_to(e2[:, None], x2.shape), x2 / x2[2:3], axis=0).T
        if geometry == "hinf":
            par = ~np.isfinite(l).all(-1)
            if par.any():
                lh = np.cross(np.broadcast_to(e2[:, None], (3, int(par.sum()))), x2[:, par], axis=0).T
                a = np.abs(lh[:, :2])
                l[par] = lh / np.where(a > 0, a, np.inf).min(-1, keepdims=True)
        lines[n] = l
    return lines


def clip_lines(lines, xmin, xmax, ymin, ymax, eps=EPS):
    """Two endpoints of each line inside the pixel-centre rectangle, or the far sentinel.
    (epipolar.py:369-405).  Returns start [N,HW,2], end [N,HW,2], nvalid [N,HW]."""
    l0, l1, l2 = lines[..., 0], lines[..., 1], lines[..., 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        by1 = -(xmin * l0 + l2) / _sd(l1, eps)
        by2 = -(xmax * l0 + l2) / _sd(l1, eps)
        bx0 = -(ymin * l1 + l2) / _sd(l0, eps)
        bx3 = -(ymax * l1 + l2) / _sd(l0, eps)
    cand = np.stack([
        np.stack([bx0, np.full_like(bx0, ymin)], -1),
        np.stack([np.full_like(by1, xmin), by1], -1),
        np.stack([np.full_like(by2, xmax), by2], -1),
        np.stack([bx3, np.full_like(bx3, ymax)], -1)], -2)              # [N,HW,4,2]
    ok = np.stack([
        (bx0 >= xmin + eps) & (bx0 < xmax - eps),
        (by1 > ymin + eps) & (by1 <= ymax - eps),
        (by2 >= ymin + eps) & (by2 < ymax - eps),
        (bx3 > xmin + eps) & (bx3 <= xmax - eps)], -1)                  # [N,HW,4]
    nvalid = ok.sum(-1)
    # first two valid candidates in order; (>2 valid makes the reference raise at :402 —
    # defined here as "first two", SURVEY appendix A)
    order = np.argsort(~ok, axis=-1, kind="stable")
    first = np.take_along_axis(cand, order[..., 0:1, None].repeat(2, -1), axis=-2)[..., 0, :]
    second = np.take_along_axis(cand, order[..., 1:2, None].repeat(2, -1), axis=-2)[..., 0, :]
    far = np.array([xmin - FAR, ymin - FAR], dtype=lines.dtype)
    bad = (nvalid < 2)[..., None]
    start = np.where(bad, far, first)
    end = np.where(bad, far, second)
    return start, end, nvalid


def sample_locs(cfg, P_ref, P_src, H, W, K=None, dtype=np.float64, geometry="reference"):
    """Normalised grid_sample coordinates of the K samples -> [K,N,H,W,2] (x,y).
    (epipolar.py:405-415; coord2pix vision/multiview.py:159-163; normalize :25-37)."""
    K = K or cfg.EPIPOLAR.SAMPLESIZE
    P_ref = np.asarray(P_ref).astype(dtype)
    P_src = np.asarray(P_src).astype(dtype)
    xs, ys = pixel_axes(cfg, H, W, dtype)
    lines = epipolar_lines(P_ref, P_src, xs, ys, geometry)
    start, end, _ = clip_lines(lines, xs[0], xs[-1], ys[0], ys[-1], dtype(EPS))
    steps = sample_steps(K, dtype).reshape(K, 1, 1, 1)
    v = start[None] + (end - start)[None] * steps                      # image coords [K,N,HW,2]
    r = dtype(cfg.DATASETS.IMAGE_RESIZE * cfg.DATASETS.PREDICT_RESIZE)
    ds = dtype(cfg.BACKBONE.DOWNSAMPLE)
    pix = (v / r + dtype(0.5) - ds / dtype(2.0)) / ds                   # feature-pixel coords
    g = np.empty_like(pix)
    if cfg.EPIPOLAR.USE_CORRECT_NORMALIZE:
        g[..., 0] = dtype(-1.0) + dtype(2.0) * pix[..., 0] / dtype(W - 1)
        g[..., 1] = dtype(-1.0) + dtype(2.0) * pix[..., 1] / dtype(H - 1)
    else:
        g[..., 0] = dtype(-1.0) + dtype(2.0) * (pix[..., 0] + dtype(0.5)) / dtype(W)
        g[..., 1] = dtype(-1.0) + dtype(2.0) * (pix[..., 1] + dtype(0.5)) / dtype(H)
    N = P_ref.shape[0]
    return g.reshape(K, N, H, W, 2)


def de_normalize(g, H, W, correct):
    """vision/multiview.py:39-57 (numpy engine branch)."""
    out = np.empty_like(g)
    if correct:
        out[..., 0] = (g[..., 0] + 1) * (W - 1) / 2.0
        out[..., 1] = (g[..., 1] + 1) * (H - 1) / 2.0
    else:
        out[..., 0] = (g[..., 0] + 1) * W / 2.0 - 0.5
        out[..., 1] = (g[..., 1] + 1) * H / 2.0 - 0.5
    return out


# ------------------------------------------------------------------------------------------
# sampling + attention                                              (epipolar.py:188-247, 272-321)
# ------------------------------------------------------------------------------------------
def grid_sample_bilinear(feat, g, align_corners=False, dtype=np.float32):
    """F.grid_sample(feat[None].expand(K), g) with mode=bilinear, padding_mode=zeros
    (epipolar.py:199,210; ATen GridSampler: unnormalize then 4 taps, OOB taps weigh 0).
    feat [C,H,W]; g [K,H,W,2] -> [K,C,H,W]."""
    C, H, W = feat.shape
    gx = g[..., 0].astype(dtype)
    gy = g[..., 1].astype(dtype)
    if align_corners:
        ix = (gx + dtype(1)) / dtype(2) * dtype(W - 1)
        iy = (gy + dtype(1)) / dtype(2) * dtype(H - 1)
    else:
        ix = ((gx + dtype(1)) * dtype(W) - dtype(1)) / dtype(2)
        iy = ((gy + dtype(1)) * dtype(H) - dtype(1)) / dtype(2)
    x0 = np.floor(ix); y0 = np.floor(iy)
    x1 = x0 + 1; y1 = y0 + 1
    w_nw = (x1 - ix) * (y1 - iy)
    w_ne = (ix - x0) * (y1 - iy)
    w_sw = (x1 - ix) * (iy - y0)
    w_se = (ix - x0) * (iy - y0)
    out = np.zeros((g.shape[0], C) + g.shape[1:3], dtype=dtype)
    featd = feat.astype(dtype)
    for xx, yy, ww in ((x0, y0, w_nw), (x1, y0, w_ne), (x0, y1, w_sw), (x1, y1, w_se)):
        inb = (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
        xi = np.clip(xx, 0, W - 1).astype(np.int64)
        yi = np.clip(yy, 0, H - 1).astype(np.int64)
        vals = featd[:, yi, xi]                                         # [C,K,H,W]
        out += np.where(inb, ww, dtype(0))[:, None] * vals.transpose(1, 0, 2, 3)
    return out


def fuse_item(feat_ref, feat_src, g, scale, align_corners=False, dtype=np.float32):
    """One (ref,src) pair given sample locations g [K,H,W,2].
    sim = sum_c samp*ref (epipolar.py:295); sim==0 -> -1e10 (:298); *scale (:306);
    softmax over K (:307); out = sum_k samp*sim (:243).  -> out [C,H,W], attn [K,H,W]."""
    samp = grid_sample_bilinear(feat_src, g, align_corners, dtype)       # [K,C,H,W]
    sim = (samp * feat_ref.astype(dtype)[None]).sum(1)                    # [K,H,W]
    sim = np.where(sim == 0, dtype(MASKED), sim) * dtype(scale)
    sim = sim - sim.max(0, keepdims=True)
    e = np.exp(sim)
    attn = e / e.sum(0, keepdims=True)
    out = (samp * attn[:, None]).sum(0)
    return out.astype(dtype), attn.astype(dtype)


def z_epilogue(out, params, zresidual, bn_eps=1e-5):
    """finalout = BN_eval(conv1x1_z(out)) [+ out]  (epipolar.py:249-253; BN.py:59-82 eval)."""
    N, C, H, W = out.shape
    Wz = np.asarray(params["z.weight"], dtype=np.float64).reshape(-1, C)
    y = np.einsum("oc,nchw->nohw", Wz, out.astype(np.float64)) + np.asarray(params["z.bias"], np.float64)[None, :, None, None]
    inv = np.asarray(params["bn.weight"], np.float64) / np.sqrt(np.asarray(params["bn.running_var"], np.float64) + bn_eps)
    y = (y - np.asarray(params["bn.running_mean"], np.float64)[None, :, None, None]) * inv[None, :, None, None] \
        + np.asarray(params["bn.bias"], np.float64)[None, :, None, None]
    if zresidual:
        y = y + out
    return y.astype(out.dtype)


def forward(cfg, feat_ref, feat_src, P_ref, P_src, params=None, locs=None, align_corners=False,
            geometry="reference", geom_dtype=np.float32, dtype=np.float32):
    """Restatement of Epipolar.forward for ATTENTION=avg, SIMILARITY=dot, SOFTMAX_ENABLED
    (epipolar.py:82-269).  Returns dict(out, attn [N,K,H,W], corr_pos [N,H,W,2], sample_locs)."""
    N, C, H, W = feat_ref.shape
    K = cfg.EPIPOLAR.SAMPLESIZE
    if locs is None:
        locs = sample_locs(cfg, P_ref, P_src, H, W, K, geom_dtype, geometry)
    locs = np.asarray(locs).astype(np.float32)                          # epipolar.py:183 .float()
    outs, attns, corrs = [], [], []
    for n in range(N):
        o, a = fuse_item(feat_ref[n], feat_src[n], locs[:, n], cfg.EPIPOLAR.SOFTMAXSCALE, align_corners, dtype)
        idx = a.argmax(0)                                               # epipolar.py:237
        pos = np.take_along_axis(locs[:, n], idx[None, :, :, None].repeat(2, -1), axis=0)[0]
        corrs.append(de_normalize(pos, H, W, cfg.EPIPOLAR.USE_CORRECT_NORMALIZE))   # :241
        outs.append(o); attns.append(a)
    out = np.stack(outs)
    if "z" in cfg.EPIPOLAR.PARAMETERIZED:
        assert params is not None
        out = z_epilogue(out, params, cfg.EPIPOLAR.ZRESIDUAL)
    return {"out": out, "attn": np.stack(attns), "corr_pos": np.stack(corrs).astype(np.float32),
            "sample_locs": locs}
