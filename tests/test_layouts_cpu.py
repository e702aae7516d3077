"""CPU: what the ABI does with the alignment of the caller's pointers, without touching a GPU.

  - The pipelined kernel writes a channels-last `out` directly with 16-byte stores only when `out` itself is 16-byte aligned;
    any other `out` takes the pixel-major plane and the transposition pass (one more region in the workspace).
  - sample_locs_in, sample_locs_out and corr_pos are read and written as (x, y) float pairs: a pointer that is not 8-byte
    aligned is refused with EPI_EINVAL before anything is launched.
  - The Python host side copies a misaligned sample_locs_in (a contiguous view at an odd element) into an aligned tensor.

The pointers below are plain integers: the size queries never dereference them, and every forward / backward call here is
refused by validation or by the workspace check before any launch."""
import ctypes

import pytest
import torch

from epipolar_transformers_b200 import _lib, build
from epipolar_transformers_b200.epipolar import _aligned_locs

ALIGNED = 256


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def align_up(v, a=256):
    return (v + a - 1) // a * a


def fwd_params(N, C, H, W, K, out=ALIGNED, channels_last_out=True):
    p = _lib.EpiFusionParams()
    p.N, p.C, p.H, p.W, p.K = N, C, H, W, K
    p.feat_ref = p.feat_src = p.P_ref = p.P_src = ALIGNED
    p.ref_stride = p.src_stride = (ctypes.c_int64 * 4)(C * H * W, H * W, W, 1)
    p.out = out
    p.out_stride = (ctypes.c_int64 * 4)(*((H * W * C, 1, W * C, C) if channels_last_out else (C * H * W, H * W, W, 1)))
    p.downsample, p.img_scale, p.eps, p.softmax_scale = 4.0, 1.0, 1e-3, 0.125
    return p


# (N, C, H, W, K): an odd map (H·W = 273) and the production shape
@pytest.mark.parametrize("shape", [(2, 64, 13, 21, 16), (4, 256, 64, 64, 64)], ids=["13x21_c64", "64x64_c256"])
def test_misaligned_out_takes_the_transposition_pass(lib, shape):
    """The same channels-last strides: at 256 and 272 (16-byte aligned) the fused kernel writes `out`; at 260 the plan adds
    the fp32 pixel-major plane (rounded up to 256 bytes) for the transposition pass."""
    N, C, H, W, K = shape
    ws = {}
    for addr in (256, 260, 264, 272):
        p = fwd_params(N, C, H, W, K, out=addr)
        assert lib.epi_fusion_cache_bytes(ctypes.byref(p)) > 0, "the pipelined kernel must be planned"
        ws[addr] = lib.epi_fusion_workspace_bytes(ctypes.byref(p))
    plane = align_up(N * C * H * W * 4)
    assert ws[272] == ws[256]
    assert ws[260] == ws[256] + plane
    assert ws[264] == ws[256] + plane                    # 8-byte aligned is not enough for a 16-byte store
    # an NCHW `out` always takes the pass, whatever its alignment
    nchw = lib.epi_fusion_workspace_bytes(ctypes.byref(fwd_params(N, C, H, W, K, out=256, channels_last_out=False)))
    assert nchw == ws[260]


@pytest.mark.parametrize("field", ["sample_locs_in", "sample_locs_out", "corr_pos"])
def test_misaligned_pair_buffers_are_refused(lib, field):
    """A pointer 4 bytes off an 8-byte boundary gives EPI_EINVAL naming the requirement; the same params with that pointer
    aligned get past validation (to the workspace check, which refuses the missing workspace: still nothing launched)."""
    N, C, H, W, K = 2, 64, 13, 21, 16
    for addr, want in ((ALIGNED + 4, -1), (ALIGNED + 8, -2)):
        p = fwd_params(N, C, H, W, K)
        setattr(p, field, addr)
        if field == "sample_locs_in":
            p.P_ref = p.P_src = None
        assert lib.epi_fusion_forward_f32(ctypes.byref(p), None) == want, (field, addr, lib.epi_last_error())
        if want == -1:
            assert b"8-byte aligned" in lib.epi_last_error()
        else:
            assert b"workspace too small" in lib.epi_last_error()


def test_misaligned_locations_refused_by_backward_and_geometry(lib):
    b = _lib.EpiFusionBwdParams()
    b.N, b.C, b.H, b.W, b.K = 2, 64, 13, 21, 16
    b.feat_ref = b.feat_src = b.attn = b.grad_out = b.grad_src = ALIGNED
    b.sample_locs_in = ALIGNED + 4
    assert lib.epi_fusion_backward_f32(ctypes.byref(b), None) == -1
    assert b"8-byte aligned" in lib.epi_last_error()
    b.sample_locs_in = ALIGNED + 8                       # aligned: refused only for the missing workspace
    assert lib.epi_fusion_backward_f32(ctypes.byref(b), None) == -2
    assert lib.epi_sample_locs_f32(ALIGNED, ALIGNED, ALIGNED + 4, 2, 13, 21, 16, 4.0, 1.0, 1e-3, 0, None) == -1
    assert b"8-byte aligned" in lib.epi_last_error()


def test_aligned_locs_copies_an_odd_offset_view():
    K, N, H, W = 3, 2, 5, 7
    flat = torch.randn(1 + K * N * H * W * 2)
    view = flat[1:].view(K, N, H, W, 2)
    assert view.is_contiguous() and view.data_ptr() % 8 == 4     # .contiguous() would hand this view on unchanged
    got = _aligned_locs(view)
    assert got.data_ptr() % 8 == 0 and got.is_contiguous()
    assert torch.equal(got, view)
    aligned = torch.randn(K, N, H, W, 2)
    assert _aligned_locs(aligned) is aligned                      # an aligned contiguous tensor is not copied
