"""Developer tool: per-phase cycles of the pipelined fused kernel (library built with `build(timers=True)`, -DEPI_PIPE_TIMERS).

Runs the cfg2 forward (N=4 pairs, C=256, 64x64, K=64, z + ZRESIDUAL, fp32) through one module, so the module's persistent
FusionState keeps the work-item records cached as in the benchmark, and prints the cycles of thread 0 of each role per work
item, summed over the CTAs.  `python tools/gpu_pipe_timers.py [H] [K] [C]`."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from epipolar_transformers_b200 import _lib
_lib.LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "libepipolar_b200_timers.so")
import epipolar_transformers_b200 as epi
from epipolar_transformers_b200 import synthetic as syn

H = int(sys.argv[1]) if len(sys.argv) > 1 else 64
K = int(sys.argv[2]) if len(sys.argv) > 2 else 64
C = int(sys.argv[3]) if len(sys.argv) > 3 else 256
N, W, CALLS = 4, H, 20
lib = _lib.load()
cfg = epi.cfg_h36m_r50_256()
cfg.KEYPOINT.HEATMAP_SIZE, cfg.KEYPOINT.NFEATS, cfg.EPIPOLAR.SAMPLESIZE = (H, W), C, K
m = epi.Epipolar(cfg=cfg).cuda().eval()
m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.z_bn_params(C).items()}, strict=False)
ring = syn.ring_cameras(4, 4 * H)
take = np.arange(N) % 4
P1 = torch.from_numpy(ring[take].astype(np.float32)).cuda()
P2 = torch.from_numpy(ring[syn.nearest_source(ring)[take]].astype(np.float32)).cuda()
g = torch.Generator(device="cuda"); g.manual_seed(1234)
f1 = torch.relu(torch.randn(N, C, H, W, device="cuda", generator=g))
f2 = torch.relu(torch.randn(N, C, H, W, device="cuda", generator=g))

timers = (ctypes.c_ulonglong * 32)()
with torch.no_grad():
    for _ in range(3):                                   # warm-up; the first call builds the cached work records
        m(f1, f2, P1, P2)
    torch.cuda.synchronize()
    lib.epi_pipe_timers_read(timers, 1)
    for _ in range(CALLS):
        m(f1, f2, P1, P2)
    torch.cuda.synchronize()
lib.epi_pipe_timers_read(timers, 1)
cta = (ctypes.c_ulonglong * 1024)()
lib.epi_pipe_cta_read(cta)                               # the last call only

v = np.array(list(timers), dtype=np.float64)
items = v[8]
print("N=%d C=%d %dx%d K=%d  calls=%d  items=%d (%.1f per call)" % (N, C, H, W, K, CALLS, items, items / CALLS))
worker = [(0, "wait for the item's descriptor"), (1, "descriptor release"), (2, "(between 1 and 3)"), (3, "GEMM1 incl. stage waits"),
          (4, "interpolation"), (5, "softmax + beta scatter"), (6, "arg-max"), (7, "beta panels"), (9, "GEMM2 + epilogue")]
tot = sum(v[s] for s, _ in worker)
print("workers (thread 0), cycles per item:")
for s, nm in worker:
    print("  slot %2d  %-34s %9.0f  %5.1f%%" % (s, nm, v[s] / items, 100 * v[s] / tot))
print("  total                                          %9.0f" % (tot / items))
print("  GEMM1 + GEMM2/epilogue (slots 3 + 9): %.1f%% of the worker cycles" % (100 * (v[3] + v[9]) / tot))
print("gather (thread 0), cycles per item:")
for s, nm in ((13, "stage acquire entry / item wait"), (14, "stage free wait"), (15, "descriptor wait"), (16, "query panel wait")):
    print("  slot %2d  %-34s %9.0f" % (s, nm, v[s] / items))
print("setup (thread 0), cycles per item:")
for s, nm in ((10, "descriptor slot free wait"), (28, "claim"), (29, "pixels + line end points"), (30, "union bitmap"),
              (31, "prefix ranks"), (17, "row list"), (18, "record publish"), (11, "hand-off")):
    print("  slot %2d  %-34s %9.0f" % (s, nm, v[s] / items))

c = np.array(list(cta), dtype=np.float64).reshape(256, 4)
grid = min(torch.cuda.get_device_properties(0).multi_processor_count, 256)
c = c[:grid]
run_us = (c[:, 2] - c[:, 1]) / 1e3
print("per CTA (last call, %d CTAs): items min/median/max %d/%d/%d, time after the dependency wait min/median/max %.1f/%.1f/%.1f us"
      % (grid, c[:, 3].min(), np.median(c[:, 3]), c[:, 3].max(), run_us.min(), np.median(run_us), run_us.max()))
hist = {int(k): int((c[:, 3] == k).sum()) for k in np.unique(c[:, 3])}
print("  CTAs by item count:", hist)
