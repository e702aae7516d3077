"""Shared helpers for the parity tests."""
import json
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    d = {k: z[k] for k in z.files}
    d["meta"] = json.loads(str(d["meta"]))
    return d


def rel_max(a, b):
    """max|a-b| / max|b|  (the T1 metric of SURVEY.md section 8c)."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def px_err(locs_a, locs_b, H, W, far=50.0):
    """Max sample-location error in feature pixels over samples that are not far-sentinels in b;
    also returns whether the far-sentinel sets agree."""
    a = np.asarray(locs_a, np.float64); b = np.asarray(locs_b, np.float64)
    fa = np.abs(a).max(-1) >= far
    fb = np.abs(b).max(-1) >= far
    scale = np.array([W / 2.0, H / 2.0])
    d = np.abs(a - b) * scale
    d = d[~fb & ~fa]
    return (float(d.max()) if d.size else 0.0), bool((fa == fb).all())


# ---- hand-built sample locations for the kernels' edge cases ------------------------------------------------------------
# Locations are normalised grid_sample coordinates [K,N,H,W,2] (x, y) for align_corners=False unless stated otherwise.

def dyadic_centres(size):
    """Pixels whose centre has a normalised coordinate (2i + 1) / size - 1 that is a multiple of 1/4 (exact in fp32).  Only
    sides of the form 4·odd (12, 20, 28, 36, ...) have any."""
    return [i for i in range(size) if (2 * i + 1) * 4 % size == 0]


def pix2grid(p, size):
    """feature-pixel coordinate -> normalised coordinate (align_corners=False), the inverse of grid_sample's unnormalize."""
    return (2.0 * np.asarray(p, np.float64) + 1.0) / size - 1.0


def edge_locs(K, N, H, W, seed):
    """[K,N,H,W,2] hand-built sample locations: random points in the map mixed with exact pixel centres (three zero-weight
    taps), points on the border, just beyond it and a pixel or more beyond it, and far-off points; pixel column 3 has only
    far-off samples.  Every value that is not random is a short dyadic fraction, so fp32 and fp64 find the same taps and
    the same zero weights (a tap weight of 1e-7 on one side only would flip the sim == 0 mask)."""
    rng = np.random.default_rng(seed)
    g = rng.uniform(-1, 1, size=(K, N, H, W, 2))
    kind = rng.integers(0, 4, size=(K, N, H, W))                 # 0 random, 1 pixel centre, 2 border, 3 far
    border = np.array([-1, 1, -1 + 1 / 64, 1 - 1 / 64, -1 - 1 / 32, 1 + 1 / 32, -1 - 1 / 16, 1 + 1 / 16, -1.25, 1.25])
    border_axis = rng.integers(0, 2, size=kind.shape)
    for axis, size in ((0, W), (1, H)):
        centres = pix2grid(dyadic_centres(size), size)            # multiples of 1/4
        assert centres.size
        on = kind == 1
        g[..., axis][on] = rng.choice(centres, size=on.sum())
        on = (kind == 2) & (border_axis == axis)
        g[..., axis][on] = rng.choice(border, size=on.sum())
    far = np.array([(-312.5, -312.5), (1e4, 0.25), (0.5, -700.0), (40.0, 40.0)])
    on = kind == 3
    g[on] = far[rng.integers(0, len(far), size=on.sum())]
    g[:, :, :, 3] = far[rng.integers(0, len(far), size=(K, N, H))]
    return g.astype(np.float32)


def with_ties(f1, f2, locs, seed, n_pix=8):
    """Exact ties at distinct locations (returns new f1, f2, locs and the tied pixels [(n, y, x, sample indices)]).  One
    random feature vector v is copied to four source pixels whose centres are dyadic, and becomes the query of `n_pix`
    reference pixels per item (not the all-far column 3, nor a zero query row).  Each of those pixels gets 2-4 samples at
    the exact centres of different copies, at random sample indices among its other samples: their sims are |v|², bit-
    identical in every kernel (one tap of weight 1 on identical rows).  v has 4x the scale of the other features, so any
    other sample's sim lies 4·sqrt(C) standard deviations below, and the first of the tied samples must win the arg-max."""
    rng = np.random.default_rng(seed)
    f1, f2, locs = f1.copy(), f2.copy(), locs.copy()
    K, N, H, W, _ = locs.shape
    cy, cx = dyadic_centres(H), dyadic_centres(W)
    tied = []
    for n in range(N):
        v = 4 * rng.standard_normal(f1.shape[1]).astype(np.float32)
        copies = [(cy[i], cx[j]) for i, j in zip(rng.permutation(len(cy))[:4], rng.permutation(len(cx))[:4])]
        for y, x in copies:
            f2[n, :, y, x] = v
        cand = [p for p in range(H * W) if p % W != 3 and f1[n, :, p // W, p % W].any()]
        for p in rng.choice(cand, size=n_pix, replace=False):
            y, x = divmod(int(p), W)
            f1[n, :, y, x] = v
            ks = np.sort(rng.choice(K, size=int(rng.integers(2, 5)), replace=False))
            for k, (sy, sx) in zip(ks, copies):
                locs[k, n, y, x] = (pix2grid(sx, W), pix2grid(sy, H))
            tied.append((n, y, x, ks))
    return f1, f2, locs, tied


def with_nonfinite(locs, seed, frac=0.15):
    """NaN, ±inf and ±1e30 in one or both coordinates of a fraction of the samples, and pixel (1, 1) entirely NaN.  A
    non-finite or huge location samples nothing (its sim is masked); corr_pos de-normalises the chosen sample's own value."""
    rng = np.random.default_rng(seed)
    locs = locs.copy()
    bad = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30], np.float32)
    on = rng.random(locs.shape[:-1]) < frac
    which = rng.integers(0, 3, size=locs.shape[:-1])                  # x, y or both
    vals = bad[rng.integers(0, len(bad), size=locs.shape)]
    for axis in (0, 1):
        m = on & ((which == axis) | (which == 2))
        locs[..., axis][m] = vals[..., axis][m]
    locs[:, :, 1, 1] = np.nan
    return locs


def block_locs(blocks, H, W):
    """sample locations at the middle (x0 + 0.5, y0 + 0.5) of 2x2 blocks [..., 2] (x0, y0): four taps of weight ≈ 0.25."""
    b = np.asarray(blocks, np.float64) + 0.5
    return np.stack([pix2grid(b[..., 0], W), pix2grid(b[..., 1], H)], -1)


def full_union_locs(K, H, W, x0s, y0s, seed):
    """[K,1,H,W,2]: every reference pixel samples K distinct blocks (x0 in x0s, y0 in y0s) at their middles.  With disjoint
    blocks one pixel's union is exactly 4K source pixels, and two different draws exceed it."""
    rng = np.random.default_rng(seed)
    blocks = np.array([(x, y) for y in y0s for x in x0s])
    pick = np.argsort(rng.random((H * W, len(blocks))), axis=1)[:, :K]     # K distinct blocks per pixel
    g = block_locs(blocks[pick], H, W)                                   # [HW,K,2]
    return np.ascontiguousarray(g.transpose(1, 0, 2).reshape(K, 1, H, W, 2)).astype(np.float32)


def wide_map_locs(K=64, H=130, W=136, seed=0):
    """Full unions on a map above 16384 pixels, where the pipelined kernel compacts the union bitmap into WIN_WORDS = 256
    (row, 32-pixel word) pairs.  Blocks have x0 in {31, 95} (each footprint row straddles the word pair 0|1 or 2|3) and rows
    (2b, 2b + 1), so each sample adds four (row, word) pairs holding one union pixel each.
      rows < H // 2: every pixel draws K = 64 distinct blocks: 256 (row, word) pairs and 256 pixels, any two pixels exceed that,
        so every work item splits down to one pixel.
      rows >= H // 2: pixels alternate between two fixed sets A and B.  Both hold 63 blocks of rows 0..127 (none at x0 = 31
        in rows 126-127); A adds a sample on column 0 (x0 = -1) in rows 126-127, B one on column 135 (x0 = W - 1) in rows
        128-129.  A ∪ B is again 256 pixels in 256 (row, word) pairs, so these items are not split.  The last pair,
        (129, word 4), is the first pixel of B's last footprint row: the only way a rank lookup reaches the last compacted
        word (every other footprint row starts in the lower word of its pair), and the word before it is row 128's copy of
        the same column, so a lookup that stopped one word short would read the other row."""
    assert (K, H, W) == (64, 130, 136)
    rng = np.random.default_rng(seed)
    blocks = np.array([(x, y) for y in range(0, H - 1, 2) for x in (31, 95)])            # 130 blocks
    top = H // 2
    pick = np.argsort(rng.random((top * W, len(blocks))), axis=1)[:, :K]
    g = np.empty((H * W, K, 2))
    g[:top * W] = block_locs(blocks[pick], H, W)
    low = blocks[(blocks[:, 1] < 128) & ~((blocks[:, 0] == 31) & (blocks[:, 1] == 126))]
    shared = low[rng.permutation(len(low))[:63]].astype(np.float64) + 0.5                # pixel coordinates of the middles
    A = np.concatenate([shared, [(-0.5, 126.5)]])       # x = -0.5: footprint x0 = -1, only column 0 in bounds
    B = np.concatenate([shared, [(135.5, 128.5)]])      # x = 135.5: x0 = 135, only column 135 in bounds
    A, B = A[rng.permutation(K)], B[rng.permutation(K)]
    for p in range(top * W, H * W):
        s = A if p % 2 == 0 else B
        g[p] = np.stack([pix2grid(s[:, 0], W), pix2grid(s[:, 1], H)], -1)
    return np.ascontiguousarray(g.transpose(1, 0, 2).reshape(K, 1, H, W, 2)).astype(np.float32)


def stereo_rig(N, img_size, yaw=0.0):
    """(P_ref, P_src) float32 [N,3,4] with integer intrinsics (f = 25/8 · img_size, principal point at the image centre).  The
    source camera of item n sits 100 (odd n: -60) units along x from the reference camera; the two are turned by -yaw/2 and
    +yaw/2 (odd n: the opposite) about the y axis, so that the baseline leaves both image planes.  yaw = 0 is an exactly
    rectified pair whose float32 matrices are exact: both epipoles lie at infinity (e[2] == 0)."""
    f, c = img_size * 25 // 8, img_size // 2
    A = np.array([[f, 0, c], [0, f, c], [0, 0, 1]], np.float64)

    def cam(s, centre):
        R = np.array([[np.cos(s), 0, np.sin(s)], [0, 1, 0], [-np.sin(s), 0, np.cos(s)]])
        return A @ np.hstack([R, (-R @ np.array([centre, 0.0, 0.0]))[:, None]])

    P1, P2 = [], []
    for n in range(N):
        s = (yaw if n % 2 == 0 else -yaw) / 2
        P1.append(cam(-s, 0.0))
        P2.append(cam(s, 100.0 if n % 2 == 0 else -60.0))
    return np.stack(P1).astype(np.float32), np.stack(P2).astype(np.float32)


# ---- camera rigs whose epipoles lie inside the maps ----------------------------------------------------------------------
# 64x64 maps of 256-pixel images (downsample 4, img_scale 1): pixel centres at 4i + 1.5, i < 64.  Cameras are built in float64
# as KRT = K [R | -R C] and cast to float32 as the dataset code does; centres and intrinsics are dyadic where a case needs exact
# arithmetic.
RIG_HW = 64


def _cam(pp, R, C, f=256.0):
    px, py = (pp, pp) if np.isscalar(pp) else pp
    A = np.array([[f, 0, px], [0, f, py], [0, 0, 1.0]])
    R = np.asarray(R, np.float64)
    return A @ np.hstack([R, (-R @ np.asarray(C, np.float64))[:, None]])


def _rot_y(a):
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])


_FLIP = np.diag([-1.0, 1.0, -1.0])                 # looking down −z: a turn by π about y, exact
_R90 = np.array([[0, 0, 1.0], [0, 1, 0], [-1, 0, 0]])   # looking down −x: a turn by −π/2 about y, exact


def ring_opposite(N=2, img=256, seed=0):
    """[V=4,N,3,4] float32: a jittered ring of 4·N cameras, view v of item n is camera v·N + n (as the views tests build it),
    so views v and v + 2 of an item are opposite cameras, both of whose epipoles lie inside the map."""
    from epipolar_transformers_b200 import synthetic as syn
    return syn.ring_cameras(4 * N, img, seed=seed, jitter=20.0).reshape(4, N, 3, 4).astype(np.float32)


def _pair_rigs():
    """name -> (P_ref [3,4], P_src [3,4]) float64 before the cast.  The reference camera's principal point is a pixel centre
    (129.5) or the centre of the map (127.5); the source camera's, (131.25, 126.125), is no pixel centre, so that no epipolar line
    through e2 meets a corner of the pixel-centre rectangle (a line through a corner is clipped on the thresholds themselves)."""
    I, pp2 = np.eye(3), (131.25, 126.125)
    return {
        # two cameras on the z axis looking at each other, the reference principal point on the centre of pixel (32, 32):
        # e1 is that pixel
        "facing": (_cam(129.5, I, (0, 0, -1024)), _cam(pp2, _FLIP, (0, 0, 1024))),
        # the same with the source centre off the axis: e1 lies between pixel centres
        "facing_off": (_cam(129.5, I, (0, 0, -1024)), _cam(pp2, _FLIP, (7, -5, 1024))),
        # the source camera behind the reference camera, looking the same way: e1's third coordinate is negative
        "behind": (_cam(129.5, I, (0, 0, -1024)), _cam(pp2, I, (0, 0, -2048))),
        "behind_off": (_cam(129.5, I, (0, 0, -1024)), _cam(pp2, _rot_y(0.02), (37, 21, -2048))),
        # facing cameras whose e1 is the centre of the pixel-centre rectangle, (127.5, 127.5), between four pixels: the
        # point the staging kernel's order key measures from
        "centre": (_cam(127.5, I, (0, 0, -1024)), _cam(pp2, _FLIP, (0, 0, 1024))),
        # the source camera turned by exactly 90°: M's third row, (−1/256, 0, 129.5/256) in fp32, depends on the reference
        # intrinsics only, so zz == 0 on all of column 32 (x = 129.5), whose rays are parallel to the source image plane
        "rig90": (_cam(129.5, I, (0, 0, -2000)), _cam(pp2, _R90, (1000, 0, 1000))),
        # its near-degenerate twin: turned by a further 1e-6 rad, zz is tiny but not zero
        "rig90_twin": (_cam(129.5, I, (0, 0, -2000)), _cam(pp2, _R90 @ _rot_y(1e-6), (1000, 0, 1000))),
    }


PAIR_RIGS = list(_pair_rigs())


def pair_rig(name):
    """-> (P_ref, P_src) float32 [N,3,4].  'ring_opposite': the 4·N opposite pairs (v, v + 2) of ring_opposite(N=2), pair
    v·N + n; otherwise one of PAIR_RIGS (N = 1)."""
    if name == "ring_opposite":
        P = ring_opposite()
        return P.reshape(-1, 3, 4), P[[2, 3, 0, 1]].reshape(-1, 3, 4)
    P1, P2 = _pair_rigs()[name]
    return P1[None].astype(np.float32), P2[None].astype(np.float32)


def epipoles(P1, P2):
    """fp64 homogeneous epipoles of one pair: e1 = P1·[C2; 1] (in the reference view), e2 = P2·[C1; 1] (in the source view)."""
    P1, P2 = np.asarray(P1, np.float64), np.asarray(P2, np.float64)
    c1 = -np.linalg.solve(P1[:, :3], P1[:, 3]); c2 = -np.linalg.solve(P2[:, :3], P2[:, 3])
    return P1 @ np.r_[c2, 1.0], P2 @ np.r_[c1, 1.0]


def img2feat(v, downsample=4.0):
    """image coordinate -> feature-pixel coordinate (img_scale 1)"""
    return (np.asarray(v, np.float64) + 0.5 - downsample / 2) / downsample


def e1_distance(P1, P2, H, W, downsample=4.0):
    """[N,H,W] distance in feature px of every reference pixel centre from e1 (inf where e1 is at infinity)."""
    d = np.empty((len(P1), H, W))
    for n in range(len(P1)):
        e1, _ = epipoles(P1[n], P2[n])
        with np.errstate(divide="ignore", invalid="ignore"):
            ex, ey = img2feat(e1[:2] / e1[2], downsample)
        d[n] = np.hypot(np.arange(W)[None, :] - ex, np.arange(H)[:, None] - ey)
    return np.nan_to_num(d, nan=np.inf)


def rig_cfg(K, C=8, H=RIG_HW, W=RIG_HW):
    from epipolar_transformers_b200.config import make_cfg
    return make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True))


def loc2feat(locs, H, W):
    """normalised (USE_CORRECT_NORMALIZE) locations [..., 2] -> feature px"""
    g = np.asarray(locs, np.float64)
    return np.stack([(g[..., 0] + 1) * (W - 1) / 2, (g[..., 1] + 1) * (H - 1) / 2], -1)


# ---- float64 reference on given locations ------------------------------------------------------------------------------
FAR_LOC = -312.5          # stands in for a non-finite location in the reference's sampling (it samples nothing either way)


def fp64_reference(f1, f2, locs, scale, correct, align_corners=False, pixels=None, chunk=512):
    """oracle.epipolar_oracle's grid_sample_bilinear / fuse_item in float64 on the fp32 locations [K,N,H,W,2], first-maximum
    arg-max, corr_pos de-normalised from the chosen sample's own fp32 value.  pixels: optional [N,P] linear pixel indices
    (the whole source map and the queries at those pixels are used), evaluated `chunk` pixels at a time.
    -> out [N,C,P], attn [N,K,P], corr [N,P,2]  (P = H·W without `pixels`)."""
    from oracle import epipolar_oracle as eo
    K, N, H, W, _ = locs.shape
    if pixels is None:
        pixels = np.broadcast_to(np.arange(H * W), (N, H * W))
    outs, attns, corrs = [], [], []
    for n in range(N):
        o_n, a_n = [], []
        for s in range(0, pixels.shape[1], chunk):
            ys, xs = np.divmod(pixels[n, s:s + chunk], W)
            g = locs[:, n, ys, xs].astype(np.float64)                              # [K,P,2]
            g[~np.isfinite(g).all(-1)] = FAR_LOC
            o, a = eo.fuse_item(f1[n][:, ys, xs][:, None], f2[n], g[:, None], scale, align_corners, np.float64)
            o_n.append(o[:, 0]); a_n.append(a[:, 0])
        o, a = np.concatenate(o_n, 1), np.concatenate(a_n, 1)
        ys, xs = np.divmod(pixels[n], W)
        pos = locs[a.argmax(0), n, ys, xs]                                           # first maximum, like torch.argmax
        outs.append(o); attns.append(a); corrs.append(eo.de_normalize(pos, H, W, correct))
    return np.stack(outs), np.stack(attns), np.stack(corrs)


# ---- a test-local driver of the C ABI ------------------------------------------------------------------------------------
# Fills EpiFusionParams / EpiFusionBwdParams from tensors the test owns, the way epipolar_fusion and epipolar_fusion_backward
# do, so that a test decides every buffer: its strides, its base address, what it holds before the call and what lies
# around it.  None of these helpers allocates an output, and none keeps a tensor alive: the caller holds every tensor it
# passes until `launch` has returned (a temporary freed earlier can be handed out again as the workspace).

def _ptr(t):
    return None if t is None else t.data_ptr()


def _strides(t):
    import ctypes
    return (ctypes.c_int64 * 4)(*(t.stride() if t is not None else (0, 0, 0, 0)))


def _feat_dtype(t):
    import torch
    from epipolar_transformers_b200 import _lib
    return {torch.float32: _lib.EPI_DTYPE_F32, torch.bfloat16: _lib.EPI_DTYPE_BF16, torch.float16: _lib.EPI_DTYPE_F16}[t.dtype]


def fusion_params(f1, f2, out, *, K, P1=None, P2=None, locs_in=None, attn=None, corr=None, locs_out=None, z=None,
                  z_residual=False, add_ref=False, variant="auto", n_src=0, align_corners=False, correct=True, downsample=4.0,
                  img_scale=1.0, scale=0.125):
    """EpiFusionParams of one forward: f1 [N,C,H,W], f2 / out [S·N,C,H,W] (any strides), z = (Wf, bf) or None."""
    from epipolar_transformers_b200 import _lib
    p = _lib.EpiFusionParams()
    N, C, H, W = f1.shape
    p.feat_ref, p.ref_stride = f1.data_ptr(), _strides(f1)
    p.feat_src, p.src_stride = f2.data_ptr(), _strides(f2)
    p.out, p.out_stride = out.data_ptr(), _strides(out)
    p.P_ref, p.P_src, p.sample_locs_in = _ptr(P1), _ptr(P2), _ptr(locs_in)
    p.attn, p.corr_pos, p.sample_locs_out = _ptr(attn), _ptr(corr), _ptr(locs_out)
    if z is not None:
        p.z_weight_folded, p.z_bias_folded = z[0].data_ptr(), z[1].data_ptr()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.downsample, p.img_scale, p.eps, p.softmax_scale = downsample, img_scale, 1e-3, scale
    p.align_corners, p.correct_normalize = int(align_corners), int(correct)
    p.z_residual, p.add_ref_residual = int(z_residual), int(add_ref)
    p.variant = _lib.VARIANTS[variant]
    p.feat_dtype = _feat_dtype(f1)
    p.n_src = n_src
    return p


def bwd_params(f1, f2, attn, g_out, *, K, P1=None, P2=None, locs_in=None, grad_ref=None, grad_src=None, deterministic=False,
               correct=True, scale=0.125):
    """EpiFusionBwdParams of one backward (grad_keys and grad_vals on, no attention gradient)."""
    from epipolar_transformers_b200 import _lib
    b = _lib.EpiFusionBwdParams()
    N, C, H, W = f1.shape
    b.feat_ref, b.ref_stride = f1.data_ptr(), _strides(f1)
    b.feat_src, b.src_stride = f2.data_ptr(), _strides(f2)
    b.P_ref, b.P_src, b.sample_locs_in = _ptr(P1), _ptr(P2), _ptr(locs_in)
    b.attn = attn.data_ptr()
    b.grad_out, b.gout_stride = g_out.data_ptr(), _strides(g_out)
    b.grad_ref, b.gref_stride = _ptr(grad_ref), _strides(grad_ref)
    b.grad_src, b.gsrc_stride = _ptr(grad_src), _strides(grad_src)
    b.N, b.C, b.H, b.W, b.K = N, C, H, W, K
    b.downsample, b.img_scale, b.eps, b.softmax_scale = 4.0, 1.0, 1e-3, scale
    b.correct_normalize = int(correct)
    b.grad_keys = b.grad_vals = 1
    b.feat_dtype = _feat_dtype(f1)
    b.deterministic = int(deterministic)
    return b


def workspace_bytes(p):
    """the forward's workspace size for these params (a pure query: nothing is launched)"""
    import ctypes
    from epipolar_transformers_b200 import _lib
    return _lib.load().epi_fusion_workspace_bytes(ctypes.byref(p))


def launch(p, workspace=None, cache=None, backward=False):
    """Runs the forward (or backward) on the current stream with the given uint8 workspace / cache tensors (None: none) and
    synchronises.  -> number of kernels launched."""
    import ctypes
    import torch
    from epipolar_transformers_b200 import _lib
    lib = _lib.load()
    if workspace is not None:
        p.workspace, p.workspace_bytes = workspace.data_ptr(), workspace.numel()
    if cache is not None:
        p.cache, p.cache_bytes = cache.data_ptr(), cache.numel()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if backward:
        _lib.check(lib.epi_fusion_backward_f32(ctypes.byref(p), stream), "epi_fusion_backward_f32")
    else:
        _lib.check(lib.epi_fusion_forward_f32(ctypes.byref(p), stream), "epi_fusion_forward_f32")
    torch.cuda.synchronize()
    return lib.epi_last_launch_count()


def corr_close(a, b):
    """corr_pos equality: 1e-4 feature px, relaxed by 1e-6 relative for the de-normalised far / huge locations (whose fp32 ulp
    exceeds it); NaN equals NaN and inf equals inf."""
    return np.isclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=1e-6, atol=1e-4, equal_nan=True).all(-1)


def check_corr(got, ref_corr, ref_attn, locs_px, H, W, correct, near=1e-6):
    """Every pixel's correspondence must be the reference's (the first maximum of the fp64 attention).  A different sample is
    accepted only at a near-tie of the fp64 attention (relative gap below `near`, not zero): exact ties must go to the first
    index.  got / ref_corr [P,2]; ref_attn [K,P]; locs_px [K,P,2] the fp32 locations.  Returns the number of near-ties."""
    from oracle import epipolar_oracle as eo
    bad = np.nonzero(~corr_close(got, ref_corr))[0]
    n_near = 0
    for i in bad:
        cand = eo.de_normalize(locs_px[:, i], H, W, correct)
        ks = np.nonzero(corr_close(cand, got[i][None]))[0]
        assert ks.size, "pixel %d: correspondence %s is not one of its samples" % (i, got[i])
        a = ref_attn[:, i]
        kr = int(a.argmax())
        ok = [k for k in ks if a[k] != a[kr] and abs(a[k] - a[kr]) < near * a[kr]]
        assert ok, "pixel %d: sample %s chosen, reference's first maximum is %d (attn %s vs %.17g)" % (
            i, ks.tolist(), kr, a[ks].tolist(), a[kr])
        n_near += 1
    return n_near
