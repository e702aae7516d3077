"""TEST INFRASTRUCTURE — freezes the byte counts the C ABI plans (epi_fusion_workspace_bytes, epi_fusion_cache_bytes,
epi_fusion_backward_workspace_bytes) over a sweep of params as tests/golden/plan_sizes.npz.  Regenerate it only when a change
to the plan is intended:
    python -m oracle.make_golden_plan [--lib path/to/libepipolar_b200.so]
The rows are enumerated by `rows()` (also used by tests/test_abi_cpu.py).  No GPU is needed: the queries read shapes only."""
from __future__ import annotations

import argparse
import ctypes
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from epipolar_transformers_b200 import _lib  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "plan_sizes.npz")
N = 2
ADDR = 256                     # stands for every device pointer: 256-byte aligned, never dereferenced by the queries

# (variant, feat_dtype, z, cache, n_src, src channels_last, out channels_last, C, (H, W), K, sample_locs_in).  C covers
# multiples of 64 (the tensor-core z GEMM) and other multiples of 8, C % 8 != 0 and C above the tile / pipe limits.  A
# channels_last output also adds the reference residual, which decides the fp32 reference copy of the fp32 z epilogue.
AXES = (range(5), range(3), (0, 1), (0, 1), (0, 1, 3), (0, 1), (0, 1), (12, 64, 256, 264, 512, 520),
        ((32, 32), (64, 64), (128, 128), (128, 256)), (16, 64, 128), (0, 1))
# invalid params: overrides of one valid row (the queries answer for them without validating)
INVALID = ({"N": 0}, {"C": 0}, {"H": 0}, {"W": -1}, {"n_src": -1}, {"variant": 7}, {"variant": -1}, {"feat_dtype": 5},
           {"K": 0}, {"K": 300}, {"C": 2000}, {"H": 1}, None)


def rows():
    return list(itertools.product(*AXES))


def _strides(C, H, W, channels_last):
    return (ctypes.c_int64 * 4)(*((H * W * C, 1, W * C, C) if channels_last else (C * H * W, H * W, W, 1)))


def _params(row, **override):
    variant, dtype, z, cache, n_src, src_cl, out_cl, C, (H, W), K, locs = row
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.variant, p.feat_dtype, p.n_src = variant, dtype, n_src
    p.feat_ref = p.feat_src = p.out = p.P_ref = p.P_src = ADDR
    p.ref_stride = _strides(C, H, W, False)
    p.src_stride = _strides(C, H, W, src_cl)
    p.out_stride = _strides(C, H, W, out_cl)
    p.add_ref_residual = out_cl
    if z:
        p.z_weight_folded = p.z_bias_folded = ADDR
    if cache:
        p.cache = ADDR
    if locs:
        p.sample_locs_in = ADDR
    for k, v in override.items():
        setattr(p, k, v)
    b = _lib.EpiFusionBwdParams()
    b.N, b.C, b.H, b.W, b.K, b.feat_dtype = p.N, p.C, p.H, p.W, p.K, p.feat_dtype
    return p, b


def sizes(lib):
    """[len(rows()) + len(INVALID), 3] uint64: forward workspace, cache, backward workspace bytes per row"""
    out = []
    for row in rows():
        p, b = _params(row)
        out.append((lib.epi_fusion_workspace_bytes(ctypes.byref(p)), lib.epi_fusion_cache_bytes(ctypes.byref(p)),
                    lib.epi_fusion_backward_workspace_bytes(ctypes.byref(b))))
    base = (_lib.EPI_VARIANT_AUTO, _lib.EPI_DTYPE_F32, 1, 0, 0, 0, 0, 256, (64, 64), 64, 0)
    for ov in INVALID:
        if ov is None:                                              # null params
            out.append((lib.epi_fusion_workspace_bytes(None), lib.epi_fusion_cache_bytes(None), lib.epi_fusion_backward_workspace_bytes(None)))
            continue
        p, b = _params(base, **ov)
        out.append((lib.epi_fusion_workspace_bytes(ctypes.byref(p)), lib.epi_fusion_cache_bytes(ctypes.byref(p)),
                    lib.epi_fusion_backward_workspace_bytes(ctypes.byref(b))))
    return np.array(out, dtype=np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="library to record from (default: the in-tree build)")
    args = ap.parse_args()
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    table = sizes(_lib.load())
    np.savez_compressed(GOLDEN, sizes=table)
    print("%s: %d rows, %d distinct workspace sizes" % (GOLDEN, len(table), len(np.unique(table[:, 0]))))


if __name__ == "__main__":
    main()
