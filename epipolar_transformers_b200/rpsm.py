"""3-D poses from the views' heat-maps on the GPU: the reference's KEYPOINT.TRIANGULATION = 'rpsm' mode, the recursive
pictorial-structure model (modeling/pictorial_cuda.py, called from modeling/model.py).

The reference runs one frame at a time: a grid_sample per view and joint, a dense 4096 x 4096 product per edge of the tree,
a copy to the host per tree node, and ten more such passes on 8 bins per joint.  Here a whole batch of frames runs in
2 + (tree depth) launches with no host synchronisation (csrc/epi_rpsm.cu), so the eval step can stay inside a CUDA graph.
The arithmetic, operation by operation, is in that file's header; oracle/rpsm_oracle.py restates it.  No CPU fallback.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib

# The reference's HumanBody (modeling/layers/body.py): root, rhip, rkne, rank, lhip, lkne, lank, belly, neck, nose, head,
# lsho, lelb, lwri, rsho, relb, rwri
H36M_PARENTS = (-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15)


def _edges(parents):
    parents = [int(p) for p in parents]
    return parents, [(parents[j], j) for j in range(len(parents)) if parents[j] != -1]


def limb_lengths(pose, parents=H36M_PARENTS):
    """pose [..., J, 3] -> [..., E] float32: the fp64 length of each edge (parent, child), edge e being the e-th non-root
    joint, as the reference's compute_limb_length, rounded once to float32 (the precision the model compares it in)."""
    _, edges = _edges(parents)
    if isinstance(pose, torch.Tensor):
        p = pose.detach().to(torch.float64)
        return torch.stack([(p[..., a, :] - p[..., c, :]).norm(dim=-1) for a, c in edges], -1).to(torch.float32)
    p = np.asarray(pose, np.float64)
    return np.stack([np.linalg.norm(p[..., a, :] - p[..., c, :], axis=-1) for a, c in edges], -1).astype(np.float32)


def crop_affine(center, scale, image_size):
    """get_affine_transform(center, scale, 0, image_size) of the reference (data/transforms/image.py) without cv2:
    center [..., 2], scale [..., 2] or [...] (×200 px) -> [..., 2, 3] float64, the affine taking the crop's three float32
    source points to its three destination points, solved in float64 as cv2.getAffineTransform does."""
    center = np.asarray(center, np.float64)
    scale = np.asarray(scale, np.float64)
    if scale.shape == center.shape[:-1]:
        scale = np.stack([scale, scale], -1)
    src_w = scale[..., 0] * 200.0
    dst_w, dst_h = float(image_size[0]), float(image_size[1])
    src = np.zeros(center.shape[:-1] + (3, 2), np.float32)
    dst = np.zeros(center.shape[:-1] + (3, 2), np.float32)
    src[..., 0, :] = center
    src[..., 1, 0] = center[..., 0]
    src[..., 1, 1] = center[..., 1] + src_w * -0.5
    dst[..., 0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[..., 1, :] = np.array([dst_w * 0.5, dst_h * 0.5]) + np.array([0, dst_w * -0.5], np.float32)
    for pts in (src, dst):                                     # get_3rd_point, in float32
        d = pts[..., 0, :] - pts[..., 1, :]
        pts[..., 2, :] = pts[..., 1, :] + np.stack([-d[..., 1], d[..., 0]], -1).astype(np.float32)
    A = np.concatenate([src.astype(np.float64), np.ones(src.shape[:-1] + (1,))], -1)              # [..., 3, 3]
    return np.swapaxes(np.linalg.solve(A, dst.astype(np.float64)), -1, -2)                       # [..., 2, 3]


def rpsm_pairwise(mask=None, limb_length=None, nbins=16, grid_size=2000.0, tolerance=150.0, parents=H36M_PARENTS, device=None):
    """The level-0 pairwise term, packed once per model: int32 [E, B, ceil(B/32)] on the GPU (B = nbins^3; bit k of row p set
    when parent bin p may take child bin k).  Give one of
      mask         the reference's PAIRWISE_FILE: a {(parent, child): [B, B]} dict (the pickle's matrices, `.todense()`) or an
                   [E, B, B] array/tensor in edge order; every entry must be 0 or 1
      limb_length  [E] limb lengths (mm): the mask is computed on the device on the level-0 grid centred at the origin, with
                   the recursions' rule |dist + 1e-9 - limb_length| < tolerance
    Runs once per model; with `mask` it checks the entries on the host."""
    lib = _lib.load()
    _lib.require_rpsm(lib)
    if (mask is None) == (limb_length is None):
        raise ValueError("give exactly one of mask and limb_length")
    parents, edges = _edges(parents)
    E = len(edges)
    if not 2 <= nbins <= _lib.RPSM_MAX_NBINS:
        raise ValueError("nbins must be in [2, %d] (got %d)" % (_lib.RPSM_MAX_NBINS, nbins))
    B = nbins ** 3
    if device is None:
        device = next((t.device for t in (mask, limb_length) if isinstance(t, torch.Tensor) and t.is_cuda),
                      torch.device("cuda", torch.cuda.current_device()))
    if mask is not None:
        if isinstance(mask, dict):
            missing = [e for e in edges if e not in mask]
            if missing:
                raise ValueError("mask has no matrix for the edges %s" % missing)
            mask = np.stack([np.asarray(mask[e], np.float32) for e in edges]) if E else np.zeros((0, B, B), np.float32)
        m = torch.as_tensor(mask).to(device=device, dtype=torch.float32).contiguous()
        if tuple(m.shape) != (E, B, B):
            raise ValueError("mask must be [E, B, B] = %s (got %s)" % ((E, B, B), tuple(m.shape)))
        if not bool(((m == 0) | (m == 1)).all()):
            raise ValueError("mask entries must be 0 or 1")
        dense, limb = m, None
    else:
        limb = torch.as_tensor(limb_length).to(device=device, dtype=torch.float32).contiguous()
        if tuple(limb.shape) != (E,):
            raise ValueError("limb_length must be [E] = [%d] (got %s)" % (E, tuple(limb.shape)))
        dense = None
    out = torch.empty((E, B, (B + 31) // 32), device=device, dtype=torch.int32)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        _lib.check(lib.epi_rpsm_pairwise_pack(dense.data_ptr() if dense is not None else None,
                                              limb.data_ptr() if limb is not None else None, E, nbins, float(grid_size),
                                              float(tolerance), out.data_ptr(), ctypes.c_void_p(stream)), "epi_rpsm_pairwise_pack")
    return out


def rpsm_views(heat, P, crop, image_size, root, limb_length, pairwise, *, parents=H36M_PARENTS, grid_size=2000.0,
               recur_nbins=2, recur_depth=10, tolerance=150.0, align_corners=False):
    """heat [V,N,J,h,w], P [V,N,3,4], crop [V,N,2,3], root [N,3], limb_length [N,E], pairwise (rpsm_pairwise) -> pose [N,J,3]
    float32 (mm).

    The layout is `triangulate_views`': per view, per frame.  heat is the `[:, 0]` slice of `forward_views(..., head=)`'s
    output mapped to the tree's joints; P the original image's cameras (origK @ RT); crop the crop affine of each view
    (crop_affine(crop_center, crop_scale, image_size)); image_size the network input (IMAGE_SIZE, x then y); root the centre
    of the level-0 cube; limb_length the recursions' limb lengths (limb_lengths()).  The level-0 cube has FIRST_NBINS = the
    pairwise term's nbins per axis and side grid_size; then recur_depth recursions with recur_nbins per axis.  Inputs of
    other float dtypes are read as float32.  One call on the current stream; never synchronises."""
    lib = _lib.load()
    _lib.require_rpsm(lib)
    named = (("heat", heat), ("P", P), ("crop", crop), ("root", root), ("limb_length", limb_length))
    for name, t in named:
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise ValueError("%s must be a floating-point tensor" % name)
    if heat.dim() != 5:
        raise ValueError("heat must be [V,N,J,h,w] (got %s)" % (tuple(heat.shape),))
    V, N, J, h, w = heat.shape
    parents, edges = _edges(parents)
    E = len(edges)
    if len(parents) != J:
        raise ValueError("parents names %d joints, heat has J = %d" % (len(parents), J))
    for name, t, shape in (("P", P, (V, N, 3, 4)), ("crop", crop, (V, N, 2, 3)), ("root", root, (N, 3)),
                           ("limb_length", limb_length, (N, E))):
        if tuple(t.shape) != shape:
            raise ValueError("%s must be %s (got %s)" % (name, shape, tuple(t.shape)))
    if not isinstance(pairwise, torch.Tensor) or pairwise.dtype != torch.int32 or pairwise.dim() != 3 or pairwise.shape[0] != E:
        raise ValueError("pairwise must be rpsm_pairwise()'s int32 [E, B, ceil(B/32)] tensor, E = %d" % E)
    B = pairwise.shape[1]
    nbins = round(B ** (1.0 / 3.0))
    if nbins ** 3 != B or pairwise.shape[2] != (B + 31) // 32:
        raise ValueError("pairwise must be [E, nbins^3, ceil(nbins^3/32)] (got %s)" % (tuple(pairwise.shape),))
    if not 2 <= V <= _lib.RPSM_MAX_VIEWS:
        raise ValueError("need 2 to %d views (got V = %d)" % (_lib.RPSM_MAX_VIEWS, V))
    if N < 1 or not 1 <= J <= _lib.RPSM_MAX_JOINTS:
        raise ValueError("need N >= 1 and 1 <= J <= %d (got N = %d, J = %d)" % (_lib.RPSM_MAX_JOINTS, N, J))
    for name, v in (("grid_size", grid_size), ("tolerance", tolerance), ("image_size[0]", image_size[0]),
                    ("image_size[1]", image_size[1])):
        if not (math.isfinite(float(v)) and float(v) > 0):
            raise ValueError("%s must be finite and positive (got %r)" % (name, v))
    if not (heat.is_cuda and P.is_cuda and crop.is_cuda and root.is_cuda and limb_length.is_cuda and pairwise.is_cuda):
        raise RuntimeError("the inputs must be CUDA tensors: the rpsm kernels have no CPU implementation")
    devs = {t.device for _, t in named} | {pairwise.device}
    if len(devs) != 1:
        raise ValueError("the inputs must be on one device (got %s)" % sorted(map(str, devs)))
    dev = heat.device
    ts = [t.detach().to(torch.float32).contiguous() for _, t in named]
    pose = torch.empty((N, J, 3), device=dev, dtype=torch.float32)
    par = (ctypes.c_int32 * J)(*parents)
    p = _lib.EpiRpsmParams()
    p.heat, p.P, p.crop, p.root, p.limb_length = (t.data_ptr() for t in ts)
    pw = pairwise.contiguous()
    p.pairwise, p.parents, p.pose = pw.data_ptr(), par, pose.data_ptr()
    p.V, p.N, p.J, p.h, p.w = V, N, J, h, w
    p.first_nbins, p.recur_nbins, p.recur_depth, p.align_corners = nbins, int(recur_nbins), int(recur_depth), int(bool(align_corners))
    p.image_size[0], p.image_size[1] = float(image_size[0]), float(image_size[1])
    p.grid_size, p.tolerance = float(grid_size), float(tolerance)
    nbytes = lib.epi_rpsm_workspace_bytes(ctypes.byref(p))
    ws = torch.empty(max(nbytes, 1), device=dev, dtype=torch.uint8)
    p.workspace, p.workspace_bytes = ws.data_ptr(), nbytes
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.epi_rpsm_f32(ctypes.byref(p), ctypes.c_void_p(stream)), "epi_rpsm_f32")
    return pose
