"""One camera view per GPU: the only exchange step of the path (SURVEY.md 8e).

The reference shards the batch with single-process nn.DataParallel (/root/reference/modeling/model.py:44) and
has no process groups.  Here every rank owns one view (its backbone output `feat_view [B,C,H,W]` for B frames and
its `KRT [3,4]`), the ranks all-gather the feature maps over NCCL/NVLink, and each rank fuses its view against
the map of its source view — the nearest camera centre, /root/reference/vision/multiview.py:59-83 and
data/datasets/multiview_h36m.py:231-238 (TOPK=1) — with the single-GPU fused kernel.  No other collective exists
on this path: pairs and pixels are independent.
"""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np
import torch
import torch.distributed as dist

from .multiview import nearest_view_table


def source_view_table(KRT_all) -> np.ndarray:
    """src(v) for every view: nearest other camera centre.  KRT_all: [V,3,4] (numpy or tensor, any device)."""
    return nearest_view_table(KRT_all, topk=1)[:, 0].astype(np.int64)


class ViewParallelFusion:
    """Holds the gather buffer and the static pairing; call once per step.

    fuse_fn(feat_ref, feat_src, P_ref, P_src) -> anything; defaults to the Epipolar sampler passed in.
    The pairing table is computed once on the host from the KRTs (they are per-camera constants in the
    reference's datasets), so the per-step path contains no host synchronisation.
    """

    def __init__(self, KRT_all, sampler: Optional[Callable] = None, group=None, fuse_fn: Optional[Callable] = None,
                 exchange: str = "p2p", sync: str = "signal"):
        """exchange='peer': the per-view maps live in symmetric (peer-mapped) memory and the fused kernels read the
        source view's map straight out of the neighbour GPU's HBM over NVLink — no copy, no collective, one
        pairwise device-side signal per step (sync='barrier' restores the all-ranks barrier); exchange='p2p': NCCL send/recv permutation (each rank receives only its
        source view's map); exchange='allgather': every rank receives all maps (what BASELINE config 4 names and
        what MULTITEST-style all-neighbour fusion needs)."""
        if exchange not in ("p2p", "allgather", "peer"):
            raise ValueError(exchange)
        self.exchange = exchange
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        KRT_all = torch.as_tensor(np.asarray(KRT_all), dtype=torch.float32)
        if KRT_all.shape[0] != self.world:
            raise ValueError("need one KRT per rank (got %d for world size %d)" % (KRT_all.shape[0], self.world))
        self.src_of = source_view_table(KRT_all)
        self.src = int(self.src_of[self.rank]) if self.world > 1 else 0
        self.consumers = [r for r in range(self.world) if int(self.src_of[r]) == self.rank and r != self.rank] if self.world > 1 else []
        self._recv = None
        self.KRT_all = KRT_all
        self.fuse_fn = fuse_fn if fuse_fn is not None else sampler
        if self.fuse_fn is None:
            raise ValueError("sampler or fuse_fn required")
        self._buf = None
        self._P_cache = {}
        self.sync = sync if sync in ("signal", "barrier") else "signal"     # peer mode: pairwise signals | full barrier

    def gather(self, feat_view: torch.Tensor) -> torch.Tensor:
        """all-gather of the per-view feature maps -> [V,B,C,H,W] (NVLink/NVSwitch under NCCL)."""
        if self.world == 1:
            return feat_view.unsqueeze(0)
        shape = (self.world * feat_view.shape[0],) + tuple(feat_view.shape[1:])      # concatenated along dim 0
        if self._buf is None or tuple(self._buf.shape) != shape or self._buf.device != feat_view.device:
            self._buf = torch.empty(shape, device=feat_view.device, dtype=feat_view.dtype)
        dist.all_gather_into_tensor(self._buf, feat_view.contiguous(), group=self.group)
        return self._buf.view((self.world,) + tuple(feat_view.shape))

    # ---- exchange='peer': symmetric memory -------------------------------------------------------------------
    def alloc_view_buffers(self, shape, dtype=torch.float32, device=None, count: int = 2):
        """`count` peer-mapped buffers for this rank's feature map (the backbone should write its output here)."""
        import torch.distributed._symmetric_memory as symm
        device = torch.device(device if device is not None else ("cuda", torch.cuda.current_device()))
        group = self.group if self.group is not None else dist.group.WORLD
        self._symm_bufs, self._symm_hdls = [], []
        for _ in range(count):
            t = symm.empty(*shape, dtype=dtype, device=device)
            self._symm_hdls.append(symm.rendezvous(t, group))
            self._symm_bufs.append(t)
        self._symm_shape, self._symm_dtype, self._symm_i = tuple(shape), dtype, 0
        return self._symm_bufs

    def peer_source(self, slot: int) -> torch.Tensor:
        """Stream-ordered hand-off, then a tensor aliasing the SOURCE rank's buffer `slot` in that GPU's memory (reads of it
        travel over NVLink inside whatever kernel consumes it).  The hand-off is pairwise, not a barrier: this rank signals
        the ranks that read ITS map ("my buffer `slot` is written", ordered after everything already enqueued on the current
        stream) and waits only for the signal of its own source rank — no rank waits for a camera it does not read."""
        h = self._symm_hdls[slot]
        if self.world == 1:
            return self._symm_bufs[slot]
        if self.sync == "signal":
            for r in self.consumers:
                h.put_signal(r, channel=0)
            h.wait_signal(self.src, channel=0)
        else:
            h.barrier(channel=0)
        return h.get_buffer(self.src, self._symm_shape, self._symm_dtype)

    def fetch_source(self, feat_view: torch.Tensor) -> torch.Tensor:
        """Point-to-point exchange: receive the source view's map, send ours to the ranks that fuse against it."""
        if self.world == 1:
            return feat_view
        if self._recv is None or self._recv.shape != feat_view.shape or self._recv.device != feat_view.device:
            self._recv = torch.empty_like(feat_view)
        send = feat_view.contiguous()
        ops = [dist.P2POp(dist.irecv, self._recv, self.src, group=self.group)]
        ops += [dist.P2POp(dist.isend, send, r, group=self.group) for r in self.consumers]
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        return self._recv

    # ---- per-camera constants on the device (built once per (device, batch); no per-step host->device copy) -------------
    def _P_dev(self, which: int, B: int, dev):
        key = (which, B, str(dev))
        t = self._P_cache.get(key)
        if t is None:
            t = self.KRT_all[which].to(dev).unsqueeze(0).expand(B, 3, 4).contiguous()
            self._P_cache[key] = t
        return t

    def P_ref_dev(self, B, dev):
        return self._P_dev(self.rank, B, dev)

    def P_src_dev(self, B, dev):
        return self._P_dev(self.src, B, dev)

    def __call__(self, feat_view: torch.Tensor, slot=None):
        """One step: exchange, then fuse this rank's view against its source view.  slot: which peer-mapped buffer
        `feat_view` is (exchange='peer'; default = round robin, with a local copy if it is not one of them)."""
        B = feat_view.shape[0]
        if self.exchange == "peer":
            if getattr(self, "_symm_bufs", None) is None or self._symm_shape != tuple(feat_view.shape):
                self.alloc_view_buffers(feat_view.shape, feat_view.dtype, feat_view.device)
            if slot is None:
                slot = self._symm_i % len(self._symm_bufs)
                self._symm_i += 1
            slot = slot % len(self._symm_bufs)
            if feat_view.data_ptr() != self._symm_bufs[slot].data_ptr():
                self._symm_bufs[slot].copy_(feat_view)          # backbone did not write in place: one local copy
            feat_src = self.peer_source(slot)
        elif self.exchange == "p2p":
            feat_src = self.fetch_source(feat_view)
        else:
            feat_src = self.gather(feat_view)[self.src]
        dev = feat_view.device
        return self.fuse_fn(feat_view, feat_src, self._P_dev(self.rank, B, dev), self._P_dev(self.src, B, dev))
