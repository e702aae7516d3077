"""Host-buffer front end of the fusion layer: pinned host tensors in, pinned host tensors out.

The reference's test loop moves every batch host->device before the model call and the predictions back
afterwards (engine/tester.py:131-134, modeling/model.py:282-300 of the original project).  The PCIe copies of the fused
layer's operands take longer than its kernels, so this class overlaps consecutive steps on two
CUDA streams — host->device copies of step i+1 run while step i's kernels and device->host copies run — with
`depth` rotating device input buffers.  With `d2h_stream=True` the results return on a THIRD stream (the step's output
tensors are handed to it with `record_stream`), so step i+1's kernels do not queue behind step i's device->host copies;
the default keeps them on the compute stream.  Every step's copies are still issued by that step's call;
`synchronize()` drains the pipeline.
"""
from __future__ import annotations

import os

import torch


def bind_host_to_gpu(index: int = 0) -> dict:
    """Pin the calling process to the CPUs local to GPU `index` (sysfs `local_cpulist` of its PCI function) so that pinned
    host buffers allocated afterwards — and the threads that drive the copies — live on the GPU's own NUMA node.  Host memory
    one socket away costs 20-40 % of the PCIe rate (measured: 0.71 vs 0.83-1.27 ms per cfg2 step end to end).  Returns
    {"previous": affinity to restore with os.sched_setaffinity(0, ...) or None, "cpus": CPUs bound, "node": NUMA node};
    a no-op (all None) where sysfs or the PCI ids are unavailable."""
    info = {"previous": None, "cpus": None, "node": None}
    try:
        pr = torch.cuda.get_device_properties(index)
        base = "/sys/bus/pci/devices/%04x:%02x:%02x.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        cpus = set()
        for part in open(base + "/local_cpulist").read().strip().split(","):
            if "-" in part:
                a, b = part.split("-")
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        prev = os.sched_getaffinity(0)
        cpus &= prev
        if cpus and cpus != prev:
            os.sched_setaffinity(0, cpus)
            info["previous"] = prev
        info["cpus"] = len(cpus)
        try:
            info["node"] = int(open(base + "/numa_node").read().strip())
        except (OSError, ValueError):
            pass
    except (OSError, AttributeError, ValueError, RuntimeError, AssertionError):
        pass
    return info


class HostStreamer:
    def __init__(self, sampler, device=None, depth: int = 2, d2h_stream: bool = False):
        self.sampler = sampler
        self.dev = torch.device(device if device is not None else "cuda")
        self.depth = depth
        self.s_in = torch.cuda.Stream(self.dev)
        self.s_run = torch.cuda.Stream(self.dev)
        self.s_out = torch.cuda.Stream(self.dev) if d2h_stream else self.s_run
        self._slots = [None] * depth
        self._free = [torch.cuda.Event() for _ in range(depth)]      # slot's device inputs may be overwritten
        self._i = 0

    def _slot(self, k, ref, src, P1, P2):
        s = self._slots[k]
        if s is None or s["ref"].shape != ref.shape:
            s = {"ref": torch.empty(ref.shape, device=self.dev, dtype=ref.dtype),
                 "src": torch.empty(src.shape, device=self.dev, dtype=src.dtype),
                 "P1": torch.empty(P1.shape, device=self.dev, dtype=torch.float32),
                 "P2": torch.empty(P2.shape, device=self.dev, dtype=torch.float32)}
            self._slots[k] = s
        return s

    def __call__(self, h_ref, h_src, h_P1, h_P2, h_out, h_attn=None, h_corr=None):
        """Enqueue one step.  h_* are pinned CPU tensors; outputs are filled asynchronously."""
        k = self._i % self.depth
        self._i += 1
        s = self._slot(k, h_ref, h_src, h_P1, h_P2)
        with torch.cuda.stream(self.s_in):
            self.s_in.wait_event(self._free[k])
            s["ref"].copy_(h_ref, non_blocking=True); s["src"].copy_(h_src, non_blocking=True)
            s["P1"].copy_(h_P1, non_blocking=True); s["P2"].copy_(h_P2, non_blocking=True)
            ev_in = torch.cuda.Event(); ev_in.record(self.s_in)
        with torch.cuda.stream(self.s_run), torch.no_grad():
            self.s_run.wait_event(ev_in)
            out, corr, attn, _ = self.sampler(s["ref"], s["src"], s["P1"], s["P2"])
            self._free[k].record(self.s_run)
            if self.s_out is self.s_run:
                for d, t in ((h_out, out), (h_attn, attn), (h_corr, corr)):
                    if d is not None and t is not None:
                        d.copy_(t, non_blocking=True)
                return
            ev_run = torch.cuda.Event(); ev_run.record(self.s_run)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(ev_run)
            for d, t in ((h_out, out), (h_attn, attn), (h_corr, corr)):
                if d is not None and t is not None:
                    t.record_stream(self.s_out)          # the allocator must not recycle the block before the copy ran
                    d.copy_(t, non_blocking=True)

    def synchronize(self):
        self.s_in.synchronize(); self.s_run.synchronize(); self.s_out.synchronize()
