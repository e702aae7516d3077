"""GPU: the launch sequence of every forward plan.  Each path launches a known number of kernels (epi_last_launch_count, which
bench.py reports), and automatic selection gives bit for bit what forcing the kernel it should pick gives."""
import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from epipolar_transformers_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def run(variant, N=2, C=64, H=32, W=32, K=32, dtype=torch.float32, src_cl=False, out_cl=False, z=False, add_ref=False,
        locs=False):
    """one epipolar_fusion on ring cameras -> (outputs, launches)"""
    P1, P2 = syn.pairs_from_ring(N, 4 * max(H, W))
    P1, P2 = torch.from_numpy(P1.astype(np.float32)).cuda(), torch.from_numpy(P2.astype(np.float32)).cuda()
    f1 = torch.from_numpy(syn.features(N, C, H, W, "randn", 1)).cuda().to(dtype)
    f2 = torch.from_numpy(syn.features(N, C, H, W, "randn", 2)).cuda().to(dtype)
    if src_cl:
        f2 = f2.contiguous(memory_format=torch.channels_last)
    out = torch.empty(N, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last) if out_cl else None
    kw = dict(K=K, correct_normalize=True, add_ref_residual=add_ref, variant=variant, out=out, want_locs=True)
    if z:
        g = torch.Generator().manual_seed(C)
        kw["z_folded"] = ((torch.randn(C, C, generator=g) / np.sqrt(C)).cuda(), (0.1 * torch.randn(C, generator=g)).cuda())
        kw["z_residual"] = True
    if locs:
        kw["sample_locs_in"] = epi.sample_locs(P1, P2, H, W, K, correct_normalize=True)
    res = epi.epipolar_fusion(f1, f2, P1, P2, **kw)
    torch.cuda.synchronize()
    return res, _lib.load().epi_last_launch_count()


# id: (forced variant, shape / options, kernels launched)
PATHS = {
    "pipe_channels_last_out": ("pipe", dict(out_cl=True), 2),                     # staging, fused
    "pipe_nchw_out": ("pipe", dict(), 3),                                         # + output transposition
    "pipe_z_c64": ("pipe", dict(z=True), 3),                                      # staging, fused, tensor-core z GEMM
    "pipe_128x256_order_apart": ("pipe", dict(H=128, W=256, out_cl=True), 3),     # the pixel order takes a launch of its own
    "pipe_bf16_z_c72_residual": ("pipe", dict(C=72, dtype=torch.bfloat16, z=True, add_ref=True), 4),   # + fp32 reference, z epilogue
    "sector": ("sector", dict(), 4),                                              # source planes, reference planes, order, fused
    "sector_z": ("sector", dict(z=True), 5),                                      # + fp32 z epilogue
    "block_tile": ("tile", dict(), 2),                                            # source planes, fused
    "warp_channels_last_src": ("warp", dict(src_cl=True), 1),                     # reads the source in place
    "warp_nchw_src": ("warp", dict(), 2),                                         # + channels-last copy of the source
    "warp_bf16": ("warp", dict(dtype=torch.bfloat16, src_cl=True), 3),            # + fp32 copies of both maps
}


@pytest.mark.parametrize("name", list(PATHS))
def test_launch_count(name):
    variant, kw, launches = PATHS[name]
    _, n = run(variant, **kw)
    assert n == launches


# id: (shape / options, the variant automatic selection must pick, kernels launched)
AUTO = {
    "pipe": (dict(), "pipe", 3),
    "k64_128x128_corner_goes_to_sector_tiles": (dict(H=128, W=128, K=64), "sector", 4),
    "k64_256x256_corner_beyond_tile_limits_goes_to_warp": (dict(H=256, W=256, K=64), "warp", 2),
    "injected_locations_k80_goes_to_block_tiles": (dict(K=80, locs=True), "tile", 2),
    "c12_goes_to_warp": (dict(C=12, K=16), "warp", 2),
}


@pytest.mark.parametrize("name", list(AUTO))
def test_auto_equals_forced_variant(name):
    kw, variant, launches = AUTO[name]
    want, n_forced = run(variant, **kw)
    got, n_auto = run("auto", **kw)
    assert n_forced == n_auto == launches
    for what, g, w in zip(("out", "corr_pos", "attn", "sample_locs"), got, want):
        assert torch.equal(g, w), what
