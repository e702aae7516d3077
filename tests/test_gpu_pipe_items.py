"""GPU: the pipelined kernel's 64-pixel work items (maps of at most 64 pixels a side, C <= 256) against its 32-pixel items on the
same inputs.  GEMM1 sums each score over the same channels in the same order whatever the item size, and everything after it is
per pixel, so attn, corr_pos and sample_locs must be bit-identical; `out` may differ in the last bits only, because GEMM2 groups
the union rows (a 64-pixel union interleaves rows that a 32-pixel half does not use) into different k16 steps.  With z the
bound is wider: the z GEMM reads the fused feature as a bf16 (hi, lo) pair, whose residual (below 2^-17 of the value) moves by
as much when the feature's last bit does."""
import ctypes

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib, synthetic as syn
from tests.util import fp64_reference

pytestmark = pytest.mark.gpu


def force_items32(on):
    lib = _lib.load()
    lib.epi_pipe_force_items32.restype = ctypes.c_int
    lib.epi_pipe_force_items32.argtypes = [ctypes.c_int]
    assert lib.epi_pipe_force_items32(1 if on else 0) == 0


@pytest.fixture(autouse=True)
def _restore_items():
    yield
    force_items32(False)


def inputs(N, C, H, K, dtype=torch.float32, cams="ring", S=1, seed=0):
    if cams == "ring":
        KRT = syn.ring_cameras(N + S, 4 * H, seed=seed, jitter=20.0)
        P1 = KRT[:N]
        P2 = np.stack([KRT[[(n + 1 + s) % (N + S) for n in range(N)]] for s in range(S)])
    else:                                   # literal random KRTs: long lines and wide unions, items split
        rng = np.random.default_rng(seed + 31)
        P1, P2 = rng.standard_normal((N, 3, 4)), rng.standard_normal((S, N, 3, 4))
    f1 = torch.from_numpy(syn.features(N, C, H, H, "randn", seed + 1)).cuda().to(dtype)
    f2 = torch.from_numpy(syn.features(S * N, C, H, H, "randn", seed + 2)).cuda().to(dtype).reshape(S, N, C, H, H)
    P1 = torch.from_numpy(P1.astype(np.float32)).cuda()
    P2 = torch.from_numpy(P2.astype(np.float32)).cuda()
    return f1, f2, P1, P2


def run(f1, f2, P1, P2, K, items32, z=None, channels_last=False, state=None):
    force_items32(items32)
    kw = dict(K=K, correct_normalize=True, want_locs=True, variant="pipe", state=state)
    if z is not None:
        kw.update(z_folded=z, z_residual=True)
    if channels_last:
        f1 = f1.contiguous(memory_format=torch.channels_last)
        f2 = torch.stack([t.contiguous(memory_format=torch.channels_last) for t in f2])
    if f2.shape[0] == 1:
        r = epi.epipolar_fusion(f1, f2[0], P1, P2[0], **kw)
    else:
        r = epi.epipolar_fusion_multi(f1, f2, P1, P2, **kw)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in r]


def check_items(a64, a32, z):
    out64, corr64, attn64, locs64 = a64
    out32, corr32, attn32, locs32 = a32
    assert np.array_equal(attn64, attn32, equal_nan=True)
    assert np.array_equal(corr64, corr32, equal_nan=True)
    assert np.array_equal(locs64, locs32, equal_nan=True)
    scale = float(np.abs(out32).max())
    assert np.abs(out64 - out32).max() <= (2e-5 if z else 1e-6) * scale, (np.abs(out64 - out32).max(), scale)


def random_z(C, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, C, generator=g) / np.sqrt(C)).float().cuda(), (0.1 * torch.randn(C, generator=g)).float().cuda()


CASES = [  # N, C, H, K, dtype, cams, S, z, channels_last
    pytest.param(4, 256, 64, 64, torch.float32, "ring", 1, True, False, id="cfg2-z"),
    pytest.param(4, 256, 64, 64, torch.float32, "ring", 1, False, True, id="cfg2-nhwc"),
    pytest.param(4, 256, 64, 64, torch.bfloat16, "ring", 1, True, True, id="cfg2-bf16-z-nhwc"),
    pytest.param(2, 64, 64, 16, torch.float32, "ring", 1, False, False, id="K16-C64"),
    pytest.param(2, 256, 64, 128, torch.float32, "ring", 1, True, False, id="K128-C256-z"),
    pytest.param(2, 64, 64, 128, torch.bfloat16, "ring", 1, False, False, id="K128-C64-bf16"),
    pytest.param(2, 128, 48, 32, torch.float32, "randn", 1, False, False, id="randn-splits"),
    pytest.param(2, 256, 64, 64, torch.float32, "ring", 3, True, False, id="nsrc3-z"),
]


@pytest.mark.parametrize("N,C,H,K,dtype,cams,S,z,cl", CASES)
def test_items64_equal_items32(N, C, H, K, dtype, cams, S, z, cl):
    f1, f2, P1, P2 = inputs(N, C, H, K, dtype, cams, S)
    zz = random_z(C) if z else None
    a64 = run(f1, f2, P1, P2, K, False, zz, cl)
    a32 = run(f1, f2, P1, P2, K, True, zz, cl)
    check_items(a64, a32, z)


def test_items64_nsrc3_equals_separate_calls():
    f1, f2, P1, P2 = inputs(2, 256, 64, 64, S=3, seed=5)
    multi = run(f1, f2, P1, P2, 64, False)
    for s in range(3):
        one = run(f1, f2[s:s + 1], P1, P2[s:s + 1], 64, False)
        for m, o in zip(multi, one):
            got = m[:, s] if m.ndim == 6 else m[s]            # sample_locs [K,S,N,H,W,2], the rest [S,N,...]
            assert np.array_equal(got, o, equal_nan=True)


def test_items64_against_fp64():
    N, C, H, K = 2, 256, 64, 64
    f1, f2, P1, P2 = inputs(N, C, H, K, seed=7)
    out, corr, attn, locs = run(f1, f2, P1, P2, K, False)
    rng = np.random.default_rng(0)
    pixels = np.stack([rng.choice(H * H, 192, replace=False) for _ in range(N)])
    ro, ra, _ = fp64_reference(f1.cpu().numpy(), f2[0].cpu().numpy(), locs, 0.125, True, pixels=pixels)
    got_o = np.stack([out[n].reshape(C, -1)[:, pixels[n]] for n in range(N)])
    got_a = np.stack([attn[n].reshape(K, -1)[:, pixels[n]] for n in range(N)])
    assert np.abs(got_o - ro).max() <= 1e-4 * np.abs(ro).max()
    assert np.abs(got_a - ra).max() <= 1e-4


def test_cache_kept_apart_between_item_sizes():
    """One persistent state alternating between 64- and 32-pixel items: a 64-pixel record covers the cache slots of two
    32-pixel records, and neither kind is ever taken for the other or read after the other overwrote part of it, so each call
    equals a fresh one."""
    f1, f2, P1, P2 = inputs(4, 256, 64, 64, seed=9)
    fresh64, fresh32 = run(f1, f2, P1, P2, 64, False), run(f1, f2, P1, P2, 64, True)
    st = epi.FusionState()
    for items32, want in ((False, fresh64), (True, fresh32), (False, fresh64), (True, fresh32)):
        got = run(f1, f2, P1, P2, 64, items32, state=st)
        for g, w in zip(got, want):
            assert np.array_equal(g, w, equal_nan=True)
