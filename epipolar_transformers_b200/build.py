"""In-tree build of the CUDA library (sm_90a) with plain nvcc — no JIT cache, so the .so
travels with the repo snapshot.  `python -m epipolar_transformers_b200.build [--force]`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libepipolar_b200.so")
STAMP = LIB + ".flags"          # the nvcc flags LIB was built with: a library built for another architecture is rebuilt
SOURCES = ["epi_abi.cu", "epi_aux.cu", "epi_fusion_warp.cu", "epi_fusion_tile.cu", "epi_fusion_pipe.cu", "epi_fusion_bwd.cu", "epi_stage.cu", "epi_peaks.cu", "epi_zgemm.cu", "epi_umma_selftest.cu", "epi_head.cu", "epi_triangulate.cu", "epi_rpsm.cu"]
HEADERS = ["epi_common.cuh", "epi_kernels.cuh", "epi_umma.cuh", os.path.join("..", "..", "include", "epipolar_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libepipolar_b200.so")


def _flags_text() -> str:
    return " ".join(NVCC_FLAGS) + "\n"


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != _flags_text():
            return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False, timers: bool = False) -> str:
    """timers=True builds libepipolar_b200_timers.so with the in-kernel clock64 phase timers (developer tool)."""
    if not timers and not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    lib = LIB.replace(".so", "_timers.so") if timers else LIB
    for s in SOURCES:
        obj = os.path.join(CSRC, s.replace(".cu", ".timers.o" if timers else ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", obj]
        if timers:
            cmd[1:1] = ["-DEPI_PIPE_TIMERS", "-DEPI_TILE_TIMERS"]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s" % s)
    subprocess.check_call([nvcc, *NVCC_FLAGS[:2], "-shared", "-o", lib, *objs, "-lcudart"])
    if not timers:
        with open(STAMP, "w") as f:
            f.write(_flags_text())
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, timers="--timers" in sys.argv))
