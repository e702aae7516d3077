"""Synthetic multi-frame inputs for the rpsm tests: random 300 mm-limbed H36M poses seen by jittered ring rigs, their heat-maps in
each view's crop, and the crop affines."""
import numpy as np

from epipolar_transformers_b200 import synthetic as syn
from epipolar_transformers_b200.rpsm import H36M_PARENTS, crop_affine, limb_lengths

J, IMG = 17, (256, 256)


def scene(V, N, seed, h=32, w=32, kind="clean", outside=False):
    """-> dict(heat [V,N,J,h,w], P [V,N,3,4], T [V,N,2,3], root [N,3], limb [N,E], X [N,J,3]) as float32 numpy.
    kind: clean Gaussians, noisy (plus |noise|), signed (plus noise and a negative offset).  outside: the root is offset by
    up to 1.5 m, so part of the level-0 cube projects outside every view."""
    rng = np.random.default_rng(seed)
    X = np.zeros((N, J, 3))
    X[:, 0] = rng.uniform(-300, 300, (N, 3)) + [0, 0, 1000]
    for c in range(1, J):
        d = rng.standard_normal((N, 3))
        X[:, c] = X[:, H36M_PARENTS[c]] + rng.uniform(250, 350, (N, 1)) * d / np.linalg.norm(d, axis=1, keepdims=True)
    P = np.stack([syn.ring_cameras(V, 1000, jitter=20.0, seed=seed * 7919 + n) for n in range(N)], 1)        # [V,N,3,4]
    uv = np.einsum("vnrc,njc->vnjr", P, np.concatenate([X, np.ones((N, J, 1))], -1))
    uv = uv[..., :2] / uv[..., 2:]
    center = uv.mean(2) + rng.normal(0, 20, (V, N, 2))
    scale = np.ptp(uv, 2).max(-1) * rng.uniform(1.2, 1.5, (V, N)) / 200.0
    T = crop_affine(center, scale, IMG).astype(np.float32)
    a = np.einsum("vnrc,vnjc->vnjr", T.astype(np.float64), np.concatenate([uv, np.ones((V, N, J, 1))], -1))
    hm = a * np.array([w / IMG[0], h / IMG[1]])
    ys, xs = np.mgrid[0:h, 0:w]
    heat = np.exp(-((xs - hm[..., 0, None, None]) ** 2 + (ys - hm[..., 1, None, None]) ** 2) / 2.0)
    if kind == "noisy":
        heat += np.abs(rng.normal(0, 0.05, heat.shape))
    elif kind == "signed":
        heat += rng.normal(0, 0.05, heat.shape) - 0.02
    root = X[:, 0] + rng.normal(0, 30, (N, 3))
    if outside:
        root += rng.uniform(-1500, 1500, (N, 3))
    return dict(heat=heat.astype(np.float32), P=P.astype(np.float32), T=T, root=root.astype(np.float32),
                limb=limb_lengths(X), X=X)
