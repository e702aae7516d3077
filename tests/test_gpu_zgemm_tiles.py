"""GPU: the tensor-core z GEMM at the edges of its tiling (128 output channels x 256 pixels of one item per CTA).

Every call forces the pipelined kernel, behind which z + BN(eval) + ZRESIDUAL runs on the tensor-core GEMM for C % 64 == 0.
The shapes put a partial pixel tile at the end of each item (H·W not a multiple of 256, odd for the per-element store path,
a multiple of 4 for the vector path), make the whole batch smaller than one tile, and leave the last block of output channels
half empty (C = 64, 192, 320).  Each result is checked against the fp64 z epilogue of the oracle applied to the oracle's
fused feature, at the tolerance of test_gpu_parity.py."""
import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from oracle import c_oracle, epipolar_oracle as eo
from tests.util import rel_max

pytestmark = pytest.mark.gpu
TOL = 1e-4
SHAPES = {"2x13x21": (2, 13, 21), "2x20x20": (2, 20, 20), "1x12x12": (1, 12, 12)}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def fold_params(params, bn_eps=1e-5):
    s = params["bn.weight"] / np.sqrt(params["bn.running_var"] + bn_eps)
    wf = (s[:, None] * params["z.weight"].reshape(len(s), -1)).astype(np.float32)
    bf = (s * (params["z.bias"] - params["bn.running_mean"]) + params["bn.bias"]).astype(np.float32)
    return dev(wf), dev(bf)


def run(C, shape, seed, maps=torch.float32, out_dtype=torch.float32):
    """the forced pipelined call with z + ZRESIDUAL + the caller's residual, and the fp64 oracle on the same map values"""
    from epipolar_transformers_b200 import synthetic as syn
    N, H, W = shape
    K = 16
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                       EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True, PARAMETERIZED=("z",), ZRESIDUAL=True))
    P1, P2 = syn.pairs_from_ring(max(N, 2), 4 * H)             # a ring of one camera has no source view
    P1, P2 = P1[:N].astype(np.float32), P2[:N].astype(np.float32)
    t1, t2 = dev(syn.features(N, C, H, W, "randn", seed)).to(maps), dev(syn.features(N, C, H, W, "randn", seed + 1)).to(maps)
    params = syn.z_bn_params(C, seed + 2)
    outs = {}
    for od in dict.fromkeys((torch.float32, out_dtype)):
        outs[od], _, _, locs = epi.epipolar_fusion(t1, t2, dev(P1), dev(P2), K=K, correct_normalize=True, want_locs=True,
                                                   z_folded=fold_params(params), z_residual=True, add_ref_residual=True,
                                                   variant="pipe", out_dtype=od)
    torch.cuda.synchronize()
    f1, f2 = t1.float().cpu().numpy(), t2.float().cpu().numpy()
    o = c_oracle.forward(cfg, f1, f2, P1, P2, locs=locs.cpu().numpy())
    want = eo.z_epilogue(o["out"], params, True) + f1
    return outs, want


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("C", [64, 128, 192, 320, 512])
def test_zgemm_tile_edges(C, shape):
    outs, want = run(C, SHAPES[shape], 31)
    assert rel_max(outs[torch.float32].cpu().numpy(), want) < TOL


@pytest.mark.parametrize("C,shape", [(128, "2x20x20"), (192, "2x13x21"), (64, "1x12x12")])
def test_zgemm_tile_edges_bf16_out(C, shape):
    """bf16 maps (the caller's residual is read as bf16) and a bf16 `out`: the float32 result within TOL of the oracle, and the
    bf16 `out` that result rounded once"""
    outs, want = run(C, SHAPES[shape], 41, maps=torch.bfloat16, out_dtype=torch.bfloat16)
    o32, o16 = outs[torch.float32], outs[torch.bfloat16]
    assert o16.dtype == torch.bfloat16
    assert rel_max(o32.cpu().numpy(), want) < TOL
    assert torch.equal(o16, o32.to(torch.bfloat16))
