"""GPU: every output element is written, nothing outside an output or the workspace is, no result depends on what the
workspace or the outputs held before, and the inputs come back unchanged.

Outputs live inside one allocation each with a 4 KB guard on both sides; outputs and guards are filled with a NaN bit pattern
no kernel writes (0x7FBADBAD; 0x7FAB for bfloat16 and 0x7DAB for float16 gradients) and compared as integers afterwards.
Each forward runs twice, with the workspace prefilled with 0x00 bytes and then with 0xFF bytes (fixed patterns, so that a
failure reproduces exactly), and a guard behind `workspace_bytes`: the two runs must give the same bits.  The persistent
cache starts zeroed; between calls only the workspace is poisoned, and every call must equal a fresh call without a cache,
also after one pair's cameras change, two pairs swap and two pairs share cameras."""
import ctypes

import numpy as np
import pytest
import torch

from epipolar_transformers_b200 import _lib
from tests.test_gpu_layouts import SHAPES, cameras, z_weights
from tests.test_gpu_pipe_items import force_items32
from tests.test_gpu_plan import PATHS
from tests.util import bwd_params, fusion_params, launch, rel_max, workspace_bytes

pytestmark = pytest.mark.gpu
GUARD = 4096
SENTINEL = {torch.float32: (torch.int32, 0x7FBADBAD), torch.bfloat16: (torch.int16, 0x7FAB), torch.float16: (torch.int16, 0x7DAB)}


@pytest.fixture(autouse=True)
def _restore_items():
    yield
    force_items32(False)


class Guarded:
    """a [shape] tensor of `dtype` (NCHW, or channels-last strides) between two 4 KB guards of one allocation, all of it
    holding the sentinel"""

    def __init__(self, shape, dtype=torch.float32, channels_last=False):
        self.itype, self.bits = SENTINEL[dtype]
        esize = torch.finfo(dtype).bits // 8
        n = int(np.prod(shape))
        g = GUARD // esize
        self.raw = torch.full((2 * g + n,), self.bits, device="cuda", dtype=self.itype)
        body = self.raw[g:g + n].view(dtype)
        if channels_last:
            N, C, H, W = shape
            self.t = body.as_strided(shape, (H * W * C, 1, W * C, C))
        else:
            self.t = body.view(shape)
        self.g, self.n = g, n

    def check(self, what):
        r = self.raw
        assert (r[:self.g] == r[0]).all() and (r[self.g + self.n:] == r[0]).all(), "%s: a guard was written" % what
        assert not (r[self.g:self.g + self.n] == r[0]).any(), "%s: %d elements never written" % (
            what, int((r[self.g:self.g + self.n] == r[0]).sum()))


def poisoned(nbytes, fill):
    """a workspace of nbytes + a trailing guard, every byte `fill`"""
    return torch.full((nbytes + GUARD,), fill, device="cuda", dtype=torch.uint8)


def int_bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


# ---------------------------------------------------------------------------------------------------------------------
# forward cases: (variant, (N, C, H, W, K), dtype, src channels-last, out channels-last, z, add_ref, n_src, 32-pixel items)
def from_plan(name):
    variant, kw, _ = PATHS[name]
    return (variant, (2, kw.get("C", 64), kw.get("H", 32), kw.get("W", 32), 32), kw.get("dtype", torch.float32), kw.get("src_cl", False),
            kw.get("out_cl", False), kw.get("z", False), kw.get("add_ref", False), 1, False)


CASES = {name: from_plan(name) for name in PATHS}
CASES.update({
    "pipe_items64_c256": ("pipe", (2, 256, 48, 48, 32), torch.float32, False, False, True, False, 1, False),
    "pipe_items32_forced_c256": ("pipe", (2, 256, 48, 48, 32), torch.float32, False, False, True, False, 1, True),
    "pipe_nsrc3_z": ("pipe", (2, 64, 32, 32, 32), torch.float32, False, False, True, True, 3, False),
    "odd_13x21_zgemm": ("auto", SHAPES["13x21"], torch.float32, False, False, True, False, 1, False),
    "odd_31x33_unstage_bf16": ("auto", SHAPES["31x33"], torch.bfloat16, True, False, False, True, 1, False),
    "odd_15x17_zfp32_refcopy_after": ("auto", SHAPES["15x17"], torch.bfloat16, False, False, True, True, 1, False),
    "odd_161x163_order_apart": ("auto", SHAPES["161x163"], torch.float32, False, True, False, False, 1, False),
    "odd_127x129_sector": ("auto", SHAPES["127x129"], torch.float32, False, False, False, False, 1, False),
    "odd_11x13_warp_f16": ("auto", SHAPES["11x13"], torch.float16, False, False, False, True, 1, False),
})


def make_inputs(shape, dtype, src_cl, S, z, seed=0):
    N, C, H, W, K = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    f1 = torch.randn((N, C, H, W), device="cuda", generator=g).to(dtype)
    f2 = torch.randn((S * N, C, H, W), device="cuda", generator=g).to(dtype)
    if src_cl:
        f2 = f2.contiguous(memory_format=torch.channels_last)
    P1, P2 = cameras(N, H, W, S, seed)
    return dict(f1=f1, f2=f2, P1=torch.from_numpy(P1).cuda(), P2=torch.from_numpy(P2).cuda(), z=z_weights(C)[1] if z else None)


def guarded_outputs(NP, C, H, W, K, out_cl):
    return dict(out=Guarded((NP, C, H, W), channels_last=out_cl), attn=Guarded((NP, K, H, W)), corr=Guarded((NP, H, W, 2)),
                locs=Guarded((K, NP, H, W, 2)))


def run_forward(x, K, outs, variant, add_ref, S, ws_fill, cache=None, z_residual=True):
    p = fusion_params(x["f1"], x["f2"], outs["out"].t, K=K, P1=x["P1"], P2=x["P2"], attn=outs["attn"].t, corr=outs["corr"].t,
                      locs_out=outs["locs"].t, z=x["z"], z_residual=z_residual and x["z"] is not None, add_ref=add_ref,
                      variant=variant, n_src=S if S > 1 else 0)
    nbytes = workspace_bytes(p)
    ws = poisoned(nbytes, ws_fill)
    launch(p, ws, cache)
    assert (ws[nbytes:] == ws_fill).all(), "the guard behind the workspace was written"
    return {k: g.t.clone() for k, g in outs.items()}


@pytest.mark.parametrize("case", list(CASES))
def test_outputs_written_and_workspace_independent(case):
    variant, shape, dtype, src_cl, out_cl, z, add_ref, S, items32 = CASES[case]
    N, C, H, W, K = shape
    force_items32(items32)
    x = make_inputs(shape, dtype, src_cl, S, z)
    before = {k: v.clone() for k, v in x.items() if isinstance(v, torch.Tensor)}
    zb = tuple(t.clone() for t in x["z"]) if z else None
    runs = []
    for fill in (0x00, 0xFF):
        outs = guarded_outputs(S * N, C, H, W, K, out_cl)
        runs.append(run_forward(x, K, outs, variant, add_ref, S, fill))
        for k, g in outs.items():
            g.check("%s (workspace 0x%02X)" % (k, fill))
    for k in runs[0]:
        assert torch.equal(int_bits(runs[0][k]), int_bits(runs[1][k])), "%s depends on the workspace's old contents" % k
    for k, v in before.items():
        assert torch.equal(int_bits(x[k]), int_bits(v)), "input %s was modified" % k
    if z:
        assert all(torch.equal(a, b) for a, b in zip(x["z"], zb)), "the z weights were modified"


def test_injected_locations_not_modified():
    """sample_locs_in is read only, and the emitted locations are exactly the injected ones"""
    N, C, H, W, K = SHAPES["13x21"]
    x = make_inputs((N, C, H, W, K), torch.float32, False, 1, False)
    locs_in = torch.rand((K, N, H, W, 2), device="cuda") * 2 - 1
    keep = locs_in.clone()
    outs = guarded_outputs(N, C, H, W, K, False)
    p = fusion_params(x["f1"], x["f2"], outs["out"].t, K=K, locs_in=locs_in, attn=outs["attn"].t, corr=outs["corr"].t,
                      locs_out=outs["locs"].t)
    launch(p, poisoned(workspace_bytes(p), 0xFF))
    for k, g in outs.items():
        g.check(k)
    assert torch.equal(int_bits(locs_in), int_bits(keep))
    assert torch.equal(int_bits(outs["locs"].t), int_bits(keep))


# ---------------------------------------------------------------------------------------------------------------------
# persistent cache
def cache_steps(P1, P2):
    """(label, P1, P2) for N = 4 pairs: the same cameras twice (miss, hit), one slot's source camera moved, two slots swapped,
    two slots given equal cameras"""
    moved = P2.clone()
    moved[2, :, 3] += torch.tensor([25.0, -10.0, 0.5], device="cuda")
    swap = [1, 0, 2, 3]
    eq1, eq2 = P1.clone(), P2.clone()
    eq1[3], eq2[3] = P1[0], P2[0]
    return [("miss", P1, P2), ("hit", P1, P2), ("one_slot_moved", P1, moved), ("hit_after_move", P1, moved),
            ("two_slots_swapped", P1[swap].contiguous(), P2[swap].contiguous()), ("two_slots_equal", eq1, eq2)]


@pytest.mark.parametrize("shape", [(4, 64, 32, 32, 32), (4, 256, 31, 33, 64)], ids=["32x32_c64", "31x33_c256_items64"])
def test_cache_hits_and_changes_equal_fresh_calls(shape):
    N, C, H, W, K = shape
    x = make_inputs(shape, torch.float32, False, 1, False, seed=3)
    p0 = fusion_params(x["f1"], x["f2"], x["f2"].float(), K=K, P1=x["P1"], P2=x["P2"], variant="pipe")
    cbytes = _lib.load().epi_fusion_cache_bytes(ctypes.byref(p0))
    assert cbytes > 0
    cache = torch.zeros(cbytes + GUARD, device="cuda", dtype=torch.uint8)
    cache[cbytes:] = 0xA5
    for i, (label, P1, P2) in enumerate(cache_steps(x["P1"], x["P2"])):
        y = dict(x, P1=P1, P2=P2)
        fresh = run_forward(y, K, guarded_outputs(N, C, H, W, K, False), "pipe", False, 1, 0x00)
        outs = guarded_outputs(N, C, H, W, K, False)
        got = run_forward(y, K, outs, "pipe", False, 1, 0xFF if i % 2 else 0x00, cache=cache[:cbytes])
        for k, g in outs.items():
            g.check("%s (%s)" % (k, label))
        for k in fresh:
            assert torch.equal(int_bits(got[k]), int_bits(fresh[k])), "%s: %s differs from a fresh call" % (label, k)
        assert (cache[cbytes:] == 0xA5).all(), "%s: the guard behind the cache was written" % label


# ---------------------------------------------------------------------------------------------------------------------
# backward
BWD = [((2, 17, 11, 13, 40), torch.float32), ((2, 64, 13, 21, 48), torch.bfloat16), ((2, 64, 13, 21, 48), torch.float16)]


@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("need", ["both", "ref", "src"])
@pytest.mark.parametrize("shape,dtype", BWD, ids=["11x13_c17_f32", "13x21_c64_bf16", "13x21_c64_f16"])
def test_backward_gradients_written_over_poisoned_workspace(shape, dtype, need, det):
    """grad_ref / grad_src between guards of their dtype's sentinel, the workspace (deterministic accumulators and coefficients
    included) prefilled with 0xFF: every requested gradient element is written, no guard is, and the gradients equal the
    fp64 autograd restatement."""
    from tests.test_gpu_backward import reference_grads
    N, C, H, W, K = shape
    x = make_inputs((N, C, H, W, K), dtype, False, 1, False, seed=8)
    attn = torch.empty((N, K, H, W), device="cuda")
    locs = torch.empty((K, N, H, W, 2), device="cuda")
    out = torch.empty((N, C, H, W), device="cuda")
    launch(fusion_params(x["f1"], x["f2"], out, K=K, P1=x["P1"], P2=x["P2"], attn=attn, locs_out=locs),
           torch.empty(1 << 24, device="cuda", dtype=torch.uint8))
    torch.manual_seed(9)
    g_out = torch.randn((N, C, H, W), device="cuda")
    gr = Guarded((N, C, H, W), dtype) if need in ("both", "ref") else None
    gs = Guarded((N, C, H, W), dtype) if need in ("both", "src") else None
    keep = [t.clone() for t in (x["f1"], x["f2"], attn, g_out, locs)]
    b = bwd_params(x["f1"], x["f2"], attn, g_out, K=K, locs_in=locs, grad_ref=gr.t if gr else None,
                   grad_src=gs.t if gs else None, deterministic=det)
    nbytes = _lib.load().epi_fusion_backward_workspace_bytes(ctypes.byref(b))
    ws = poisoned(nbytes, 0xFF)
    launch(b, ws, backward=True)
    assert (ws[nbytes:] == 0xFF).all(), "the guard behind the backward workspace was written"
    for t, k in zip((x["f1"], x["f2"], attn, g_out, locs), keep):
        assert torch.equal(int_bits(t), int_bits(k)), "an input of the backward was modified"
    _, e1, e2 = reference_grads(x["f1"].float(), x["f2"].float(), locs, g_out, None)
    tol = 1e-4 + (torch.finfo(dtype).eps if dtype != torch.float32 else 0.0)
    for g, e, what in ((gr, e1, "grad_ref"), (gs, e2, "grad_src")):
        if g is None:
            continue
        g.check(what)
        assert rel_max(g.t.float().cpu().numpy(), e.cpu().numpy()) < tol, what
