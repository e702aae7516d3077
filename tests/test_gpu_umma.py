"""GPU: the wgmma building blocks (descriptors, 128B swizzle, accumulator fragment mapping, bf16 hi/lo split) checked as
plain GEMMs against torch fp32/fp64 matmul before the fusion kernel relies on them."""
import ctypes

import pytest
import torch

from epipolar_transformers_b200 import _lib

pytestmark = pytest.mark.gpu


def run(mode, A, B, N, K, split):
    lib = _lib.load()
    D = torch.zeros(128, N, device="cuda")
    rc = lib.epi_umma_selftest(mode, A.data_ptr(), B.data_ptr(), D.data_ptr(), N, K, split,
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    return D


@pytest.mark.parametrize("N,K", [(32, 64), (32, 256), (64, 128), (16, 256)])
@pytest.mark.parametrize("split", [0, 1])
def test_k_major(N, K, split):
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + K)
    A = torch.randn(128, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    D = run(0, A, B, N, K, split)
    if split:
        ref = (A.double() @ B.double().T).float()
        tol = 3e-5
    else:
        ref = (A.bfloat16().double() @ B.bfloat16().double().T).float()
        tol = 2e-6
    err = (D - ref).abs().max().item() / ref.abs().max().item()
    assert err < tol, err


@pytest.mark.parametrize("N,K", [(32, 64), (32, 128), (64, 128)])
@pytest.mark.parametrize("split", [0, 1])
def test_mn_major_a(N, K, split):
    g = torch.Generator(device="cuda").manual_seed(N * 77 + K)
    At = torch.randn(K, 128, device="cuda", generator=g)       # [Kd, M]
    B = torch.randn(N, K, device="cuda", generator=g)
    D = run(1, At, B, N, K, split)
    if split:
        ref = (At.double().T @ B.double().T).float()
        tol = 3e-5
    else:
        ref = (At.bfloat16().double().T @ B.bfloat16().double().T).float()
        tol = 2e-6
    err = (D - ref).abs().max().item() / ref.abs().max().item()
    assert err < tol, err
