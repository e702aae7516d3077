"""GPU: when the layer reads and writes memory, not only what it computes.

Every other test writes its inputs, makes one call and synchronises.  These run the layer the way a model does: behind
producers still in flight on its stream, ahead of consumers on the same and on other streams, call after call through one
persistent state, on several streams and host threads at once, and captured in CUDA graphs.  Every result is compared, bit for
bit, with the eager reference: the same call on the same values, run alone with a synchronise before and after.

  A. Producers in flight: a sleep, then a copy that writes input set Y into one input, then the call with no synchronise.  The
     result must be eager(Y).  Each case asserts eager(X) != eager(Y) and that the copy had not finished when the call had
     been enqueued; the sleep is at least 20x the slowest measured call, and 20 to 50 ms.  This checks stream ordering, host
     code that reads no input value and the device-side camera key; a memcpy producer cannot overlap a launch, so the
     kernels' programmatic-dependent-launch waits are exercised by B's back-to-back calls only.
  B. Consumers and the next call: outputs read on the same stream and copied on a side stream right after the call, then a run
     of calls through one FusionState (and through the module's own state) with a synchronise at the end only.
  C. A fold enqueued behind a sleep on one stream and used at once on another; two modules on two streams at once; two host
     threads with their own streams, modules and C (so their z GEMM tensor maps and attribute flags differ).
  D. CUDA graphs: capture after a side-stream warm-up (PyTorch's recipe), then replays with new features and the same cameras
     (cached pair records) and with new cameras (the device-side cache key must miss inside a replay); a captured module
     follows an in-place update of its z weights.
  E. One host thread on two devices (the kernels' shared-memory attributes are set per device).

Each plan is asserted by its launch count (epi_last_launch_count) and by whether it keeps a cache (the pipelined kernel only):
pipe + tensor-core z GEMM, pipe + fp32 z epilogue, pipe with a direct `out`, pipe + transposition pass (bf16 `out`, injected
locations), forced sector, tile and warp kernels, n_src = 3, the views form with and without a source table, and the backward
in its default and deterministic forms."""
import threading
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import _lib
from epipolar_transformers_b200.epipolar import epipolar_fusion_backward
from epipolar_transformers_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
N, H, W, K = 2, 16, 20, 32
SLEEP_MS_MIN, SLEEP_MS_MAX = 20.0, 50.0
ATOMIC_TOL = 1e-5            # the default backward's dL/dfeat_src against its eager call, relative to its largest magnitude


def launches():
    return _lib.load().epi_last_launch_count()


@dataclass(frozen=True)
class Case:
    form: str                    # single | multi | views | bwd
    C: int
    launches: int
    pipe: bool
    z: bool = False
    z_residual: bool = False
    add_ref: bool = False
    variant: str = "auto"
    channels_last: bool = False  # maps (and so `out`) channels-last: the fused kernel stores `out` itself
    out_dtype: torch.dtype = torch.float32
    locs_in: bool = False
    want_locs: bool = False
    S: int = 1                   # multi: sources per reference item
    V: int = 0                   # views: views per frame
    table: tuple = None          # views: the [V,S] source table
    deterministic: bool = False  # bwd


CASES = {
    "pipe_zgemm": Case("single", 256, 3, True, z=True, z_residual=True, add_ref=True),
    "pipe_zfp32": Case("single", 264, 3, True, z=True),
    "pipe_direct": Case("single", 64, 2, True, channels_last=True, want_locs=True),
    "pipe_unstage_bf16": Case("single", 64, 3, True, out_dtype=torch.bfloat16),
    "pipe_locs_in": Case("single", 64, 3, True, locs_in=True),
    "sector": Case("single", 64, 4, False, variant="sector"),
    "tile": Case("single", 64, 2, False, variant="tile"),
    "warp": Case("single", 64, 2, False, variant="warp"),
    "nsrc3_zgemm": Case("multi", 64, 3, True, z=True, S=3),
    "views": Case("views", 64, 3, True, V=3),
    "views_table_zgemm": Case("views", 128, 3, True, z=True, z_residual=True, V=4, table=((1, 2), (2, 3), (3, 0), (0, 1))),
    "views_table_bf16": Case("views", 64, 3, True, V=4, table=((1,), (2,), (3,), (0,)), out_dtype=torch.bfloat16),
    "bwd_default": Case("bwd", 64, 3, False),
    "bwd_deterministic": Case("bwd", 64, 5, False, deterministic=True),
}


def cameras(n_items, n_cams, seed):
    """[n_cams, n_items, 3, 4] float32: camera c of item n is view (n + c) of a jittered ring (a different ring per seed)"""
    KRT = syn.ring_cameras(n_items + n_cams, 4 * max(H, W), seed=seed, jitter=40.0)
    P = np.stack([KRT[[(n + c) % (n_items + n_cams) for n in range(n_items)]] for c in range(n_cams)])
    return torch.from_numpy(P.astype(np.float32)).cuda()


def make_inputs(name, seed):
    """one input set of case `name`: every tensor the call reads, keyed by the argument it is passed as"""
    c = CASES[name]
    g = torch.Generator().manual_seed(seed)

    def feat(*shape):
        t = torch.randn(shape, generator=g).cuda()
        return t.contiguous(memory_format=torch.channels_last) if c.channels_last else t

    d = {}
    if c.form in ("single", "bwd"):
        P = cameras(N, 2, seed)
        d.update(feat_ref=feat(N, c.C, H, W), feat_src=feat(N, c.C, H, W), P_ref=P[0], P_src=P[1])
    elif c.form == "multi":
        P = cameras(N, 1 + c.S, seed)
        d.update(feat_ref=feat(N, c.C, H, W), feat_srcs=torch.randn((c.S, N, c.C, H, W), generator=g).cuda(), P_ref=P[0],
                 P_srcs=P[1:].contiguous())
    else:
        d.update(feats=torch.randn((c.V, N, c.C, H, W), generator=g).cuda(), P=cameras(N, c.V, seed).contiguous())
    if c.locs_in:
        d["sample_locs_in"] = (torch.rand((K, N, H, W, 2), generator=g) * 2.4 - 1.2).cuda()
    if c.z:
        d["z_weight"] = (torch.randn((c.C, c.C), generator=g) / c.C ** 0.5).cuda()
        d["z_bias"] = (0.1 * torch.randn((c.C,), generator=g)).cuda()
    if c.form == "bwd":
        _, _, attn, locs = epi.epipolar_fusion(d["feat_ref"], d["feat_src"], d["P_ref"], d["P_src"], K=K, correct_normalize=True,
                                               want_locs=True)
        d.update(attn=attn, sample_locs=locs, grad_out=torch.randn((N, c.C, H, W), generator=g).cuda(),
                 grad_attn=(0.1 * torch.randn((N, K, H, W), generator=g)).cuda())
    torch.cuda.synchronize()
    return d


def varied_inputs(name):
    """the inputs of case `name` that a caller's producer may still be writing (A): the maps, the cameras (not with injected
    locations, nor in the backward, which samples at the forward's locations), the injected locations and the folded z
    weight and bias; in the backward the maps and both incoming gradients"""
    c = CASES[name]
    if c.form == "bwd":
        return ["feat_ref", "feat_src", "grad_out", "grad_attn"]
    keys = {"single": ["feat_ref", "feat_src", "P_ref", "P_src"], "multi": ["feat_ref", "feat_srcs", "P_ref", "P_srcs"],
            "views": ["feats", "P"]}[c.form]
    if c.locs_in:
        keys = [k for k in keys if not k.startswith("P")] + ["sample_locs_in"]
    return keys + (["z_weight", "z_bias"] if c.z else [])


A_PARAMS = [pytest.param(n, k, id="%s-%s" % (n, k)) for n in CASES for k in varied_inputs(n)]


def call(name, d, state=None):
    """the case's call on input set d (no synchronise) -> dict of its outputs"""
    c = CASES[name]
    if c.form == "bwd":
        g_ref, g_src = epipolar_fusion_backward(d["feat_ref"], d["feat_src"], d["P_ref"], d["P_src"], d["attn"], d["grad_out"],
                                                K=K, correct_normalize=True, grad_attn=d["grad_attn"],
                                                sample_locs_in=d["sample_locs"], deterministic=c.deterministic)
        return dict(grad_ref=g_ref, grad_src=g_src)
    kw = dict(K=K, correct_normalize=True, want_locs=c.want_locs, variant=c.variant, state=state, out_dtype=c.out_dtype,
              add_ref_residual=c.add_ref, sample_locs_in=d.get("sample_locs_in"))
    if c.z:
        kw.update(z_folded=(d["z_weight"], d["z_bias"]), z_residual=c.z_residual)
    if c.form == "single":
        r = epi.epipolar_fusion(d["feat_ref"], d["feat_src"], d["P_ref"], d["P_src"], **kw)
    elif c.form == "multi":
        r = epi.epipolar_fusion_multi(d["feat_ref"], d["feat_srcs"], d["P_ref"], d["P_srcs"], **kw)
    else:
        r = epi.epipolar_fusion_views(d["feats"], d["P"], sources=c.table, **kw)
    return {k: v for k, v in zip(("out", "corr_pos", "attn", "sample_locs"), r) if v is not None}


def eager(name, d):
    """the reference: the call alone, synchronised before and after, through a fresh state; asserts the case's plan"""
    torch.cuda.synchronize()
    state = epi.FusionState()
    r = call(name, d, state)
    torch.cuda.synchronize()
    c = CASES[name]
    assert launches() == c.launches, (name, launches())
    if c.form != "bwd":
        assert (state.cache is not None) == c.pipe, name
    return r


def bits(t):
    return t.contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()])


def assert_same(got, want, tag=""):
    assert got.keys() == want.keys(), tag
    for k in want:
        assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype, (tag, k)
        assert torch.equal(bits(got[k]), bits(want[k])), "%s: %s differs from the eager call (max |diff| %.3g)" % (
            tag, k, (got[k].double() - want[k].double()).abs().max().item())


def unordered_sum(name, k):
    """the default backward's dL/dfeat_src sums with float atomics in no fixed order (the deterministic path is the one with
    fixed bits): two runs on the same inputs may differ in the last bits"""
    c = CASES.get(name)
    return c is not None and c.form == "bwd" and not c.deterministic and k == "grad_src"


def rel_diff(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def assert_result(name, got, want, tag=""):
    """bit for bit, except an unordered sum: held to ATOMIC_TOL of its largest magnitude"""
    for k in [k for k in want if unordered_sum(name, k)]:
        err = rel_diff(got[k], want[k])
        assert err <= ATOMIC_TOL, "%s: %s differs from the eager call by %.3g (relative)" % (tag, k, err)
    assert_same({k: v for k, v in got.items() if not unordered_sum(name, k)},
                {k: v for k, v in want.items() if not unordered_sum(name, k)}, tag)


def assert_differs(a, b, keys=None, name=None):
    """detection power: the two eager results differ in every output compared (`keys`: those that can; None: all) — bit for
    bit, and an unordered sum of case `name` by more than the ATOMIC_TOL that assert_result allows it"""
    for k in keys or a:
        if unordered_sum(name, k):
            assert rel_diff(a[k], b[k]) > ATOMIC_TOL, "%s differs by no more than its run-to-run tolerance" % k
        else:
            assert not torch.equal(bits(a[k]), bits(b[k])), "%s is the same for both input sets" % k


# ---------------------------------------------------------------------------------------------------------------------
# A. producers still in flight on the same stream
@pytest.fixture(scope="session")
def sleep_cycles():
    """torch.cuda._sleep cycles for at least 20x the slowest case's call (median of five, CUDA events), and at least
    SLEEP_MS_MIN ms so that the host has enqueued the call long before the sleep ends (each test asserts that it has); at
    most SLEEP_MS_MAX ms.  Measured once per session."""
    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    worst = 0.0
    for name in CASES:
        d = make_inputs(name, 1)
        state = epi.FusionState()
        for _ in range(2):
            call(name, d, state)
        torch.cuda.synchronize()
        worst = max(worst, float(np.median([timed(lambda: call(name, d, state)) for _ in range(5)])))
    per_ms = 10 ** 7 / timed(lambda: torch.cuda._sleep(10 ** 7))
    sleep_ms = min(SLEEP_MS_MAX, max(SLEEP_MS_MIN, 20 * worst))
    assert sleep_ms >= 20 * worst, "the slowest call takes %.3f ms: 20x exceeds the %g ms bound" % (worst, SLEEP_MS_MAX)
    print("\nslowest call %.3f ms; sleep %.2f ms = %d cycles" % (worst, sleep_ms, int(sleep_ms * per_ms)))
    return int(sleep_ms * per_ms)


def differing_outputs(name, key):
    """the outputs input `key` decides (None: all of them): the maps do not move the sample locations, and the z weights
    reach `out` only (a changed map moves the correspondences only where it changes an arg-max, so they are not required to
    differ).  The backward takes the forward's attention as given, so dL/dfeat_ref does not depend on feat_ref."""
    if CASES[name].form == "bwd":
        return ["grad_src"] if key == "feat_ref" else None
    if key.startswith("P") or key == "sample_locs_in":
        return None
    return ["out"] if key.startswith("z_") else ["out", "attn"]


@pytest.mark.parametrize("name,key", A_PARAMS)
def test_producer_in_flight(name, key, sleep_cycles):
    """The layer is called while the copy that writes its input `key` still waits behind a sleep on the stream; the result
    is eager(Y), and eager(X) differs from it.  This checks stream ordering, that no input value is read on the host, and
    that the device-side camera key sees new values behind unchanged pointers (a cache miss).  It cannot check the kernels'
    programmatic-dependent-launch waits: the copy is a memcpy (and a torch kernel never triggers its dependents early), so the
    layer's first kernel starts only once it has completed.  Those waits are exercised between the layer's own calls, by B."""
    X, Y = make_inputs(name, 1), make_inputs(name, 2)
    want_x = eager(name, X)
    want_y = eager(name, dict(X, **{key: Y[key]}))
    assert_differs(want_x, want_y, differing_outputs(name, key), name)
    state = epi.FusionState()
    call(name, X, state)                      # the state holds X's plan and cached cameras: Y's cameras miss
    torch.cuda.synchronize()
    copied = torch.cuda.Event()
    torch.cuda._sleep(sleep_cycles)
    X[key].copy_(Y[key])
    copied.record()
    got = call(name, X, state)
    in_flight = not copied.query()
    torch.cuda.synchronize()
    assert in_flight, "the copy had finished before the call was enqueued: the sleep is too short to test anything"
    assert launches() == CASES[name].launches
    assert_result(name, got, want_y, "%s/%s" % (name, key))


# ---------------------------------------------------------------------------------------------------------------------
# B. consumers and the next call
SEQUENCE = (0, 0, 1, 1, 0, 0, 1, 1)          # input set per call: X, X (the cache hits), Y (misses), Y (hits), ...


@pytest.mark.parametrize("name", list(CASES))
def test_consumers_and_call_sequence(name):
    """Right after a call, a torch op on the same stream and a copy on a side stream (behind an event recorded after the call)
    read every output; then eight calls through one FusionState alternate two input sets with different cameras, each with
    outputs of its own, and the stream is synchronised once at the end.  Every result must be its eager one.

    The sequence is a regression guard: a kernel that rewrites the state's planes, pixel order or work records while the
    previous call's kernels still read them need not show in one run, and the test does not repeat it to hunt for a race."""
    X, Y = make_inputs(name, 1), make_inputs(name, 2)
    want = [eager(name, X), eager(name, Y)]
    assert_differs(*want, name=name)
    state = epi.FusionState()
    side = torch.cuda.Stream()
    r = call(name, X, state)
    same = {k: v.clone() for k, v in r.items()}
    done = torch.cuda.Event()
    done.record()
    side.wait_event(done)
    with torch.cuda.stream(side):
        other = {k: v.clone() for k, v in r.items()}
    seq = []
    for i in SEQUENCE:
        seq.append(call(name, (X, Y)[i], state))
        assert launches() == CASES[name].launches
    torch.cuda.synchronize()
    assert_result(name, same, want[0], "same stream")
    assert_result(name, other, want[0], "side stream")
    for n, (i, got) in enumerate(zip(SEQUENCE, seq)):
        assert_result(name, got, want[i], "call %d" % n)


def load_z(m, C, seed):
    """random z conv / BN parameters and statistics (syn.z_bn_params) into module m"""
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v).view(sd[k].shape) for k, v in syn.z_bn_params(C, seed).items()}, strict=False)
    return m


def z_module(C, seed):
    """an eval Epipolar with the z projection and ZRESIDUAL (cfg2's flags), the residual fused and the locations returned"""
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=C),
                       EPIPOLAR=dict(SAMPLESIZE=K, PARAMETERIZED=("z",), ZRESIDUAL=True, USE_CORRECT_NORMALIZE=True),
                       VIS=dict(EPIPOLAR_LINE=True))
    return load_z(epi.Epipolar(cfg=cfg, fuse_ref_residual=True).cuda().eval(), C, seed)


def module_inputs(C, seed, n=N, h=H, w=W):
    g = torch.Generator().manual_seed(seed)
    P = cameras(n, 2, seed)
    return dict(feat1=torch.randn((n, C, h, w), generator=g).cuda(), feat2=torch.randn((n, C, h, w), generator=g).cuda(),
                P1=P[0], P2=P[1])


def module_call(m, d):
    with torch.no_grad():
        r = m(d["feat1"], d["feat2"], d["P1"], d["P2"])
    return {k: v for k, v in zip(("out", "corr_pos", "attn", "sample_locs"), r) if v is not None}


def module_eager(m, d):
    torch.cuda.synchronize()
    r = module_call(m, d)
    torch.cuda.synchronize()
    assert launches() == 3                   # staging, fused kernel, z GEMM
    return r


def test_module_call_sequence():
    """B through the module's own state (one per stream) and its cached fold: eight calls, one synchronise."""
    m = z_module(256, 1)
    X, Y = module_inputs(256, 1), module_inputs(256, 2)
    want = [module_eager(m, X), module_eager(m, Y)]
    assert_differs(*want)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):               # a stream the module has no state on yet
        seq = [module_call(m, (X, Y)[i]) for i in SEQUENCE]
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for n, (i, got) in enumerate(zip(SEQUENCE, seq)):
        assert_same(got, want[i], "call %d" % n)


# ---------------------------------------------------------------------------------------------------------------------
# C. side streams and host threads
def test_fold_on_one_stream_first_use_on_another(sleep_cycles):
    """The module's first eval call is made on stream A behind a sleep, so its z / BN fold is enqueued there and not yet run;
    the next call, at once, is on stream B, whose inputs are ready.  B must wait for the fold (the event the fold recorded).
    The fold's buffers are placed where a NaN-filled block of the same sizes was freed on A, so a call on B that did not wait
    would read NaN: the check is deterministic."""
    C = 256
    m = z_module(C, 3)
    X, Y = module_inputs(C, 1), module_inputs(C, 2)
    ref = z_module(C, 3)
    want_a, want_b = module_eager(ref, X), module_eager(ref, Y)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        poison = (torch.full((C, C), float("nan"), device="cuda"), torch.full((C,), float("nan"), device="cuda"))
        ptrs = {t.data_ptr() for t in poison}
    torch.cuda.synchronize()
    del poison                                   # back to A's pool, NaN-filled
    folded = torch.cuda.Event()
    with torch.cuda.stream(a):
        torch.cuda._sleep(sleep_cycles)
        got_a = module_call(m, X)
        folded.record()
    assert {t.data_ptr() for t in m._fold_cache[1]} == ptrs, "the fold did not reuse the poisoned blocks"
    with torch.cuda.stream(b):
        got_b = module_call(m, Y)
    in_flight = not folded.query()
    torch.cuda.synchronize()
    assert in_flight, "the fold had run before the call on B was enqueued: the sleep is too short to test anything"
    assert_same(got_a, want_a, "stream A")
    assert_same(got_b, want_b, "stream B")


def test_concurrent_streams():
    """Two modules (z GEMM at C = 256, and no z at C = 64) run on two streams at the same time, three calls each, enqueued
    alternately; every result equals the serial run's."""
    m1 = z_module(256, 1)
    cfg = epi.make_cfg(KEYPOINT=dict(HEATMAP_SIZE=(H, W), NFEATS=64), EPIPOLAR=dict(SAMPLESIZE=K, USE_CORRECT_NORMALIZE=True))
    m2 = epi.Epipolar(cfg=cfg).cuda().eval()
    ins1 = [module_inputs(256, s) for s in (1, 2, 3)]
    ins2 = [module_inputs(64, s) for s in (4, 5, 6)]
    want1 = [module_eager(m1, d) for d in ins1]
    torch.cuda.synchronize()
    want2 = []
    for d in ins2:
        want2.append(module_call(m2, d))
        torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream()); s2.wait_stream(torch.cuda.current_stream())
    got1, got2 = [], []
    for d1, d2 in zip(ins1, ins2):
        with torch.cuda.stream(s1):
            got1.append(module_call(m1, d1))
        with torch.cuda.stream(s2):
            got2.append(module_call(m2, d2))
    torch.cuda.synchronize()
    for i in range(3):
        assert_same(got1[i], want1[i], "stream 1 call %d" % i)
        assert_same(got2[i], want2[i], "stream 2 call %d" % i)


def run_in_thread(fn, *args):
    """fn(*args) on a host thread of its own, joined before returning -> its result (its exception is re-raised here)"""
    box = {}

    def body():
        try:
            box["r"] = fn(*args)
        except BaseException as e:           # noqa: BLE001 - re-raised in the test's thread
            box["e"] = e

    t = threading.Thread(target=body)
    t.start()
    t.join()
    if "e" in box:
        raise box["e"]
    return box["r"]


def test_host_threads():
    """Two host threads, each with its own stream and module (C = 256 and 128, so the z GEMM's per-thread tensor-map cache and
    the kernels' attribute flags differ), loop four calls at the same time.  Every result equals the serial run's, and the
    launch count each thread reads is its own call's."""
    Cs = (256, 128)
    mods = [z_module(C, i) for i, C in enumerate(Cs)]
    ins = [[module_inputs(C, 10 * i + s) for s in range(4)] for i, C in enumerate(Cs)]
    want = [[module_eager(m, d) for d in ds] for m, ds in zip(mods, ins)]
    start = threading.Barrier(2)
    results, errors = [None, None], []

    def worker(i):
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.default_stream())
            got, counts = [], []
            start.wait(timeout=60)
            with torch.cuda.stream(s):
                for d in ins[i]:
                    got.append(module_call(mods[i], d))
                    counts.append(launches())
            s.synchronize()
            results[i] = (got, counts)
        except BaseException as e:          # noqa: BLE001 - reported by the test's thread
            errors.append(e)
            start.abort()

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
    assert not any(t.is_alive() for t in threads), "a worker thread did not finish"
    if errors:
        raise errors[0]
    for i in range(2):
        got, counts = results[i]
        assert counts == [3] * 4, (Cs[i], counts)
        for n in range(4):
            assert_same(got[n], want[i][n], "C=%d call %d" % (Cs[i], n))


# ---------------------------------------------------------------------------------------------------------------------
# D. CUDA-graph capture and replay
def capture(fn, warmup=3):
    """PyTorch's recipe: warm fn up on a side stream, then capture it -> (graph, its static outputs)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    torch.cuda.synchronize()
    return g, out


def replay_and_check(g, static, outs, inputs_for, ref):
    """replays with (features of a new set, the captured cameras) twice, then with a new set's cameras too; each against
    ref(the values the static inputs then hold).  inputs_for(seed, new_cameras) -> {static key: values}."""
    for seed, new_cams in ((11, False), (12, False), (13, True)):
        vals = inputs_for(seed, new_cams)
        for k, v in vals.items():
            static[k].copy_(v)
        want = ref({k: t.clone() for k, t in static.items()})
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert_same({k: v.clone() for k, v in outs.items()}, want, "replay seed %d%s" % (seed, " new cameras" if new_cams else ""))


def features_cameras(make, keys_cams):
    """inputs_for of replay_and_check for an input maker: features always new, cameras only when asked"""
    def inputs_for(seed, new_cams):
        d = make(seed)
        return {k: v for k, v in d.items() if new_cams or k not in keys_cams}
    return inputs_for


def test_graph_module_cfg2():
    """The eval module with z + ZRESIDUAL at cfg2's shape (N = 4, C = 256, 64x64, K = 64) captured after a side-stream
    warm-up, which has cached a fold: the graph makes its own fold, and waits on nothing recorded outside it."""
    cfg = epi.cfg_h36m_r50_256()
    m = load_z(epi.Epipolar(cfg=cfg).cuda().eval(), 256, 5)
    make = lambda seed: module_inputs(256, seed, n=4, h=64, w=64)
    static = make(10)
    ref_m = epi.Epipolar(cfg=cfg).cuda().eval()
    ref_m.load_state_dict(m.state_dict())
    g, outs = capture(lambda: module_call(m, static))
    assert launches() == 3
    replay_and_check(g, static, outs, features_cameras(make, ("P1", "P2")), lambda d: module_eager(ref_m, d))


def test_graph_module_follows_parameter_update():
    """A captured module folds z / BN when it replays, reading the parameters in place: after an in-place update of z.weight
    and an eager call (which re-folds and frees the fold it had cached), a replay equals the eager call on the new weights and
    differs from the result before the update."""
    m = z_module(256, 1)
    static = module_inputs(256, 10)
    g, outs = capture(lambda: module_call(m, static))
    before = module_eager(m, static)
    g.replay()
    torch.cuda.synchronize()
    assert_same({k: v.clone() for k, v in outs.items()}, before, "before the update")
    with torch.no_grad():
        m.z.weight.mul_(1.5)
    after = module_eager(m, static)
    assert_differs(before, after, keys=["out"])
    g.replay()
    torch.cuda.synchronize()
    assert_same({k: v.clone() for k, v in outs.items()}, after, "after the update")


def graph_case(name, seed0=10):
    """capture of case `name`'s call through a caller's FusionState (made on the warm-up stream, so the graph keeps its cache)"""
    static = make_inputs(name, seed0)
    state = epi.FusionState()
    g, outs = capture(lambda: call(name, static, state))
    assert launches() == CASES[name].launches
    cams = {k for k in static if k.startswith("P")}
    replay_and_check(g, static, outs, features_cameras(lambda s: make_inputs(name, s), cams), lambda d: eager(name, d))


@pytest.mark.parametrize("name", ["views_table_bf16", "pipe_direct", "pipe_zfp32", "pipe_unstage_bf16", "pipe_zgemm"])
def test_graph_replay(name):
    """The views form with a source table and a bf16 `out`, a direct pipe call with want_locs, the fp32 z epilogue and the
    transposition pass, each captured and replayed with new features (cache hits) and new cameras (a miss)."""
    graph_case(name)


def test_graph_two_calls():
    """Two back-to-back calls through one state in one graph: the second call's cameras differ from the first's, so inside
    every replay the first call's cache records are replaced by the second's and back again."""
    name = "pipe_zgemm"
    A, B = make_inputs(name, 20), make_inputs(name, 21)
    state = epi.FusionState()
    g, outs = capture(lambda: (call(name, A, state), call(name, B, state)))
    for seed in (22, 23):
        A2, B2 = make_inputs(name, seed), make_inputs(name, seed + 100)
        for k in A:
            A[k].copy_(A2[k]); B[k].copy_(B2[k])
        want = (eager(name, A2), eager(name, B2))
        g.replay()
        torch.cuda.synchronize()
        assert_same(outs[0], want[0], "first call")
        assert_same(outs[1], want[1], "second call")


# ---------------------------------------------------------------------------------------------------------------------
# E. one host thread on two devices
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_one_thread_two_devices():
    """A thread that has run the layer on cuda:0 runs it on cuda:1: every launch above 48 KB of shared memory there needs
    its attribute set on that device too.  Each device's result equals a fresh thread's run on that device."""
    def run(dev):
        with torch.cuda.device(dev):
            m = z_module(256, 1).to(dev)
            d = {k: v.to(dev) for k, v in module_inputs(256, 1).items()}
            r = module_call(m, d)
            torch.cuda.synchronize(dev)
            return {k: v.cpu() for k, v in r.items()}

    want = [run_in_thread(run, d) for d in (0, 1)]
    got = run_in_thread(lambda: [run(0), run(1)])
    for i in range(2):
        assert_same(got[i], want[i], "cuda:%d" % i)
