"""TEST INFRASTRUCTURE — numpy restatement of the recursive pictorial-structure kernels (csrc/epi_rpsm.cu), vectorised over frames.

Every float32 operation of the kernels is restated as the same IEEE operation in the same order: numpy's float32 +, -, *, /
and sqrt round once, and `fma32` rounds a*b + c once (the product is exact in float64; the float64 sum is rounded to odd
and then to float32, which is a correctly rounded fused multiply-add).  So the oracle's pose equals the kernels' bit for bit.
The reference (modeling/pictorial_cuda.py) computes the projection with BLAS matmuls in an unspecified order; the golden
file (tests/golden/rpsm.npz, made by oracle/make_golden_rpsm.py from the unmodified reference) pins this restatement to it.
"""
from __future__ import annotations

import numpy as np

H36M_PARENTS = (-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15)
f32 = np.float32


@np.errstate(all="ignore")
def fma32(a, b, c):
    """fl32(a·b + c), rounded once"""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b                                                  # exact: 24 + 24 bits
    s = p + c
    # two-sum: the exact error of s; round s to odd when it is inexact, so the float32 rounding below is the correct one
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    odd = (bits & 1) == 1
    fix = (err != 0) & ~odd & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def linspace32(size, n):
    """torch.linspace(-size/2, size/2, n) in float32 (CPU kernel: each half one fused multiply-add)"""
    start, end = f32(-size / 2), f32(size / 2)
    step = f32((end - start) / f32(n - 1))
    i = np.arange(n)
    lo = fma32(step, i.astype(np.float32), start)
    hi = fma32(-step, (n - 1 - i).astype(np.float32), end)
    return np.where(i < n // 2, lo, hi).astype(np.float32)


def level_sizes(grid_size, first_nbins, recur_nbins, depth):
    """the reference's cur_grd_size chain (Python floats): level 0, then each recursion's"""
    out, s = [float(grid_size)], float(grid_size) / first_nbins
    for _ in range(depth):
        out.append(s)
        s = s / recur_nbins
    return out


def grid_offsets(n):
    """bin b -> (ix, iy, iz), meshgrid 'ij': b = (ix·n + iy)·n + iz"""
    b = np.arange(n ** 3)
    return np.stack([b // (n * n), (b // n) % n, b % n], -1)


def grid(g, centre):
    """g [n] 1-D grid, centre [..., 3] float32 -> [..., n^3, 3]: fl(g[i] + c)"""
    idx = grid_offsets(len(g))
    return (g[idx][None] + np.asarray(centre, np.float32)[..., None, :]).astype(np.float32)


def tree(parents):
    parents = list(parents)
    J = len(parents)
    root = parents.index(-1)
    edges = [j for j in range(J) if j != root]                 # edge e = the e-th non-root joint
    depth = np.zeros(J, int)
    for j in range(J):
        k = j
        while parents[k] != -1:
            k = parents[k]
            depth[j] += 1
    children = [[c for c in range(J) if parents[c] == p] for p in range(J)]
    return dict(J=J, root=root, edges=edges, edge_of={c: e for e, c in enumerate(edges)}, depth=depth, children=children,
                parents=parents)


# ---- unary ----------------------------------------------------------------------------------------------------------------------
def grid_coords(X, P, T, image_size, h, w):
    """X [..., 3] float32 points; P [..., 3, 4], T [..., 2, 3] float32 broadcast against X's leading axes -> (gx, gy)"""
    x, y, z = X[..., 0], X[..., 1], X[..., 2]
    q = [((P[..., r, 0] * x + P[..., r, 1] * y) + P[..., r, 2] * z) + P[..., r, 3] for r in range(3)]
    u, t = q[0] / q[2], q[1] / q[2]
    a = (T[..., 0, 0] * u + T[..., 0, 1] * t) + T[..., 0, 2]
    b = (T[..., 1, 0] * u + T[..., 1, 1] * t) + T[..., 1, 2]
    a = (a * f32(w)) / f32(image_size[0])
    b = (b * f32(h)) / f32(image_size[1])
    return (a / f32(h - 1)) * f32(2) - f32(1), (b / f32(w - 1)) * f32(2) - f32(1)


def grid2pix(g, size, align):
    g1 = g + f32(1)
    return (g1 * f32(0.5)) * f32(size - 1) if align else fma32(g1, f32(size), f32(-1)) * f32(0.5)


def taps(gx, gy, h, w, align):
    """epi_common.cuh's make_taps: north-west tap, the four weights, the four in-bounds flags"""
    ix, iy = grid2pix(gx, w, align), grid2pix(gy, h, align)
    nan = np.isnan(ix) | np.isnan(iy)
    fx = np.clip(np.floor(ix), -2, w)
    fy = np.clip(np.floor(iy), -2, h)
    with np.errstate(invalid="ignore"):
        ax, ay = ix - np.floor(ix), iy - np.floor(iy)
    fx, fy = np.where(nan, -2, fx), np.where(nan, -2, fy)
    ax, ay = np.where(nan, f32(0), ax).astype(np.float32), np.where(nan, f32(0), ay).astype(np.float32)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    wts = [(f32(1) - ax) * (f32(1) - ay), ax * (f32(1) - ay), (f32(1) - ax) * ay, ax * ay]
    inb = [(x0 + dx >= 0) & (x0 + dx < w) & (y0 + dy >= 0) & (y0 + dy < h) for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1))]
    return x0, y0, wts, inb


def sample(maps, x0, y0, wts, inb):
    """maps [M, h, w] float32, tap arrays [M, K] -> [M, K]: the in-bounds taps' w·value, nw, ne, sw, se, from 0"""
    h, w = maps.shape[-2:]
    m = np.arange(maps.shape[0])[:, None]
    s = np.zeros(x0.shape, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
            yy, xx = np.clip(y0 + dy, 0, h - 1), np.clip(x0 + dx, 0, w - 1)
            s = np.where(inb[k], s + wts[k] * maps[m, yy, xx], s).astype(np.float32)
    return s


def unary(heat, P, T, image_size, X, align):
    """heat [V,N,J,h,w]; P [V,N,3,4], T [V,N,2,3]; X [N,K,3] (one grid for all joints) or [N,J,K,3] -> U [N,J,K]"""
    V, N, J, h, w = heat.shape
    shared = X.ndim == 3
    U = None
    for v in range(V):
        Pv, Tv = P[v][:, None], T[v][:, None]
        if not shared:
            Pv, Tv = Pv[:, None], Tv[:, None]
        with np.errstate(all="ignore"):
            gx, gy = grid_coords(X, Pv, Tv, image_size, h, w)
        if shared:
            gx, gy = np.broadcast_to(gx[:, None], (N, J) + gx.shape[1:]), np.broadcast_to(gy[:, None], (N, J) + gy.shape[1:])
        x0, y0, wts, inb = taps(gx.reshape(N * J, -1), gy.reshape(N * J, -1), h, w, align)
        s = sample(heat[v].reshape(N * J, h, w), x0, y0, wts, inb).reshape(N, J, -1)
        U = s if U is None else (U + s).astype(np.float32)
    return U


# ---- pairwise and max-product -----------------------------------------------------------------------------------------------------
def limb_ok(Xp, Xc, L, tol):
    """Xp [..., 3], Xc [..., 3] float32, L float32 -> bool: |fl(sqrt(n2) + 1e-9) - L| < tol"""
    d = (Xp - Xc) + f32(1e-6)
    n2 = fma32(d[..., 2], d[..., 2], fma32(d[..., 1], d[..., 1], d[..., 0] * d[..., 0]))
    dist = np.sqrt(n2) + f32(1e-9)
    return np.abs(dist - np.asarray(L, np.float32)) < f32(tol)


def pairwise_mask(limb, nbins, grid_size, tol):
    """[E, B, B] bool on the level-0 grid centred at the origin (row = parent bin)"""
    X = grid(linspace32(grid_size, nbins), np.zeros(3, np.float32))[0]
    return np.stack([limb_ok(X[:, None], X[None], f32(L), tol) for L in np.asarray(limb, np.float32)])


def golden_mask(limb, seed, nbins=16, grid_size=2000.0, tol=150.0, density=0.01):
    """the golden cases' level-0 mask: the limb-length mask, or with seed >= 0 that mask OR a random one of the given density"""
    mask = pairwise_mask(limb, nbins, grid_size, tol)
    if seed >= 0:
        mask |= np.random.default_rng(seed).random(mask.shape, np.float32) < density
    return mask


def torch_max(v, axis=-1):
    """torch.max / np.argmax on the last axis: the first NaN, else the first maximum (+0 == -0) -> (value, index)"""
    i = np.argmax(v, axis=axis)
    return np.take_along_axis(v, i[..., None], axis)[..., 0], i


def maxprod_dense(pw, Ec):
    """pw [..., P, K] float32 0/1, Ec [..., K] -> m, s [..., P]: max_k pw·E (the product in float32, 0·inf = NaN)"""
    with np.errstate(invalid="ignore"):
        return torch_max((pw * Ec[..., None, :]).astype(np.float32))


class SparseMask:
    """one edge's [B, B] mask as rows of set columns, for the level-0 max-product of many frames"""

    def __init__(self, mask):
        self.B = mask.shape[1]
        self.rows, self.cols = np.nonzero(mask)
        counts = np.bincount(self.rows, minlength=mask.shape[0])
        self.start = np.concatenate([[0], np.cumsum(counts)[:-1]])
        self.empty = counts == 0
        off = ~mask
        self.has_off = off.any(1)
        self.koff = np.where(self.has_off, off.argmax(1), 0)
        self.dense = mask.astype(np.float32)


def maxprod0(sm: SparseMask, Ec):
    """Ec [N, B] -> m, s [N, B]: torch.max over k of mask·E_c, from the set columns and the first masked-off bin when every
    E_c is finite, densely otherwise"""
    N = Ec.shape[0]
    m = np.empty((N, len(sm.empty)), np.float32)
    s = np.empty((N, len(sm.empty)), np.int64)
    fin = np.isfinite(Ec).all(1)
    for n in np.flatnonzero(~fin):
        m[n], s[n] = maxprod_dense(sm.dense, Ec[n])
    idx = np.flatnonzero(fin)
    counts = np.bincount(sm.rows, minlength=len(sm.empty))
    for c in range(0, len(idx), 16):
        nn = idx[c:c + 16]
        Ecn = Ec[nn]
        # a sentinel column behind the set columns, so every row's start is a valid reduceat index
        vals = np.concatenate([Ecn[:, sm.cols], np.full((len(nn), 1), -np.inf, np.float32)], 1)
        seg = np.maximum.reduceat(vals, sm.start, axis=1)
        rep = np.concatenate([np.repeat(seg, counts, axis=1), np.full((len(nn), 1), np.inf, np.float32)], 1)
        cols = np.concatenate([sm.cols, [sm.B]])
        first = np.minimum.reduceat(np.where(vals == rep, cols[None], sm.B), sm.start, axis=1)
        first = np.where(sm.empty, 0, first)
        on_v = np.where(sm.empty, np.float32(-np.inf), np.take_along_axis(Ecn, first, 1))
        zval = (f32(0) * Ecn[:, sm.koff]).astype(np.float32)
        take_off = sm.has_off & (sm.empty | (on_v < 0) | ((on_v == 0) & (sm.koff < first)))
        m[nn] = np.where(take_off, zval, on_v)
        s[nn] = np.where(take_off, sm.koff, first)
    return m, s


# ---- the model ------------------------------------------------------------------------------------------------------------------
def infer(U, maxprod, t):
    """U [N,J,K] unaries; maxprod(parent, child, E_child [N,K]) -> (m, s) [N,Kp] -> bins [N,J], per-edge states"""
    N = U.shape[0]
    E = U.copy()
    S = {}
    for d in range(int(t["depth"].max()), 0, -1):
        for p in range(t["J"]):
            if t["depth"][p] != d - 1 or not t["children"][p]:
                continue
            for c in t["children"][p]:
                m, S[c] = maxprod(p, c, E[:, c])
                with np.errstate(invalid="ignore", over="ignore"):
                    E[:, p] = (E[:, p] * m).astype(np.float32)
    bins = np.zeros((N, t["J"]), np.int64)
    bins[:, t["root"]] = torch_max(E[:, t["root"]])[1]
    for j in sorted(range(t["J"]), key=lambda j: t["depth"][j]):
        if j != t["root"]:
            bins[:, j] = np.take_along_axis(S[j], bins[:, t["parents"][j]][:, None], 1)[:, 0]
    return bins, E


def rpsm(heat, P, T, image_size, root, limb, mask, parents=H36M_PARENTS, grid_size=2000.0, recur_nbins=2, recur_depth=10,
         tolerance=150.0, align_corners=False, picks=False, chunk=32):
    """`rpsm_chunk` over chunks of `chunk` frames (the level-0 arrays of a whole batch would not fit in memory)"""
    N = np.shape(root)[0]
    kw = dict(parents=parents, grid_size=grid_size, recur_nbins=recur_nbins, recur_depth=recur_depth, tolerance=tolerance,
              align_corners=align_corners)
    outs = [rpsm_chunk(heat[:, a:a + chunk], P[:, a:a + chunk], T[:, a:a + chunk], image_size, root[a:a + chunk],
                       limb[a:a + chunk], mask, **kw) for a in range(0, N, chunk)]
    if not picks:
        return np.concatenate([o[0] for o in outs])
    return (np.concatenate([o[0] for o in outs]), np.concatenate([o[1] for o in outs], 1),
            [np.concatenate([o[2][r] for o in outs]) for r in range(recur_depth + 1)])


def rpsm_chunk(heat, P, T, image_size, root, limb, mask, parents=H36M_PARENTS, grid_size=2000.0, recur_nbins=2, recur_depth=10,
               tolerance=150.0, align_corners=False):
    """heat [V,N,J,h,w], P [V,N,3,4], T [V,N,2,3], root [N,3], limb [N,E] (float32), mask [E,B,B] bool -> pose [N,J,3] float32
    -> (pose, the chosen bins per level [D+1, N, J], each level's root energies)"""
    heat = np.asarray(heat, np.float32)
    P, T = np.asarray(P, np.float32), np.asarray(T, np.float32)
    root, limb = np.asarray(root, np.float32), np.asarray(limb, np.float32)
    t = tree(parents)
    n0 = round(mask.shape[1] ** (1 / 3))
    sizes = level_sizes(grid_size, n0, recur_nbins, recur_depth)
    X0 = grid(linspace32(sizes[0], n0), root)                                   # [N,B,3]
    U = unary(heat, P, T, image_size, X0, align_corners)
    sms = [SparseMask(mask[e]) for e in range(len(t["edges"]))]
    bins, E = infer(U, lambda p, c, Ec: maxprod0(sms[t["edge_of"][c]], Ec), t)
    pose = np.take_along_axis(X0, bins[..., None], 1)                           # [N,J,3]
    levels, roots = [bins], [E[:, t["root"]]]
    for r in range(recur_depth):
        X = grid(linspace32(sizes[r + 1], recur_nbins), pose)                   # [N,J,RB,3]
        U = unary(heat, P, T, image_size, X, align_corners)

        def mp(p, c, Ec, X=X):
            pw = limb_ok(X[:, p, :, None], X[:, c, None], limb[:, t["edge_of"][c], None, None], tolerance).astype(np.float32)
            return maxprod_dense(pw, Ec)
        bins, E = infer(U, mp, t)
        pose = np.take_along_axis(X, bins[..., None, None], 2)[:, :, 0]
        levels.append(bins)
        roots.append(E[:, t["root"]])
    return pose, np.stack(levels), roots

