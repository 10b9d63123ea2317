"""Host-to-host pipelining of a set-abstraction module over a large batch of clouds.

The operators launch on the *current* CUDA stream (and the FPS workspace is stream-ordered), so a
batch that lives in pinned host memory can be processed in chunks: the H2D copies of all chunks are
queued back to back on a copy stream, groups of chunks compute on one of a few compute streams as
soon as they have landed, and results return on a third stream (PCIe is full duplex).

    pipe = HostPipeline(sa_module, chunk_clouds=132, n_streams=2)
    pipe(host_feats, out_xyz_host, out_points_host)      # all pinned; returns after a full sync

For a STREAM of batches (a loader handing over one pinned batch after another) the copies of batch i+1 need not wait for batch i:

    for batch in loader:
        pipe.submit(batch, out_xyz_host, out_points_host)   # returns at once; H2D of this batch overlaps the previous batch's kernels
    pipe.drain()

``submit`` runs the module over the WHOLE batch (the kernel shapes of the device-resident path, 8 clouds per SM) from one of two
device input buffers; the copy of the next batch lands in the other one meanwhile, results return on a third stream.

``host_feats`` is the reference's model input layout ``(B, C, N)`` with xyz in channels 0..2
(``models/modules/pointnet_pp.py:43-47``: ``l0_xyz = xyz[:, :3, :]``).
"""
from __future__ import annotations

from typing import List, Sequence

import torch

from . import pointnet2_utils as pn2


class HostPipeline:
    """H2D copies run back to back on a dedicated stream in chunks of ``chunk_clouds`` into ONE device
    buffer; compute runs on ``n_streams`` streams over GROUPS of consecutive chunks (``groups``: chunks
    per group in order, the last but one repeating, the last entry being the size of the final group) as soon as the last chunk of a group has landed;
    results return on a third stream.  The kernels of a chunk are sized to own an SM (the group-MLP CTA takes all 64K
    registers, the FPS sort prologue most of the shared memory), so chunks on different streams mostly run one after the
    other and the end-to-end time is about first H2D + chunks x (compute time of one chunk)."""

    def __init__(self, module: torch.nn.Module, chunk_clouds: int = 132, n_streams: int = 2,
                 groups: Sequence[int] = (1,), fps_mode: int = None, sa_engine: int = None):
        self.module = module
        self.chunk = int(chunk_clouds)
        self.groups = tuple(int(g) for g in groups) or (1,)
        self.fps_mode = fps_mode          # None: shape by the clouds in flight; else the tgn_furthestsampling mode of every chunk
        self.sa_engine = sa_engine        # None: leave the module's engine choice; 5 = half-size group-MLP CTAs that share an SM with other chunks' kernels
        self.streams: List[torch.cuda.Stream] = [torch.cuda.Stream() for _ in range(max(1, int(n_streams)))]
        self.copy_in = torch.cuda.Stream()
        self.copy_out = torch.cuda.Stream()
        self._dev = None
        self._ring, self._ring_free, self._submitted, self._last = None, [None, None], 0, None

    def _plan(self, B: int):
        """[(lo, hi)] of the chunks and [(first_chunk, last_chunk)] of the compute groups."""
        spans = [(lo, min(B, lo + self.chunk)) for lo in range(0, B, self.chunk)]
        body, tail = self.groups[:-1], self.groups[-1]
        plan, k, i = [], 0, 0
        while k < len(spans):
            remaining = len(spans) - k
            if remaining <= tail or not body:
                n = min(remaining, tail)
            else:                                   # body entries in order, the last one repeating; keep the tail group
                n = max(1, min(body[min(i, len(body) - 1)], remaining - tail))
                i += 1
            plan.append((k, k + n - 1))
            k += n
        return spans, plan

    @torch.no_grad()
    def __call__(self, host_feats: torch.Tensor, out_xyz_host: torch.Tensor, out_points_host: torch.Tensor) -> None:
        B = host_feats.shape[0]
        main = torch.cuda.current_stream()
        if self._dev is None or self._dev.shape != host_feats.shape:
            self._dev = torch.empty(host_feats.shape, dtype=host_feats.dtype, device="cuda")
        dev = self._dev
        self.copy_in.wait_stream(main)
        self.copy_out.wait_stream(main)
        for s in self.streams:
            s.wait_stream(main)
        spans, plan = self._plan(B)
        landed = []
        with torch.cuda.stream(self.copy_in):                  # every H2D copy queued up front, back to back
            for lo, hi in spans:
                dev[lo:hi].copy_(host_feats[lo:hi], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self.copy_in)
                landed.append(ev)
        saved_mode, saved_engine = pn2._fps_mode, pn2._sa_engine
        if self.sa_engine is not None:
            pn2.set_sa_engine(self.sa_engine)
        for gi, (k0, k1) in enumerate(plan):
            lo, hi = spans[k0][0], spans[k1][1]
            s = self.streams[gi % len(self.streams)]
            s.wait_event(landed[k1])
            # FPS shape for the clouds resident on the GPU (this group and its neighbour on the other stream)
            pn2.set_fps_mode(self.fps_mode if self.fps_mode is not None else 0)      # 0: the library picks by the clouds of the call
            with torch.cuda.stream(s):
                d = dev[lo:hi]
                new_xyz, new_points = self.module(d[:, :3].contiguous(), d)
                if not new_xyz.is_contiguous():        # the modules return the reference's permuted view of (B,S,3)
                    new_xyz = pn2.transpose_last2(new_xyz.permute(0, 2, 1))
                done = torch.cuda.Event()
                done.record(s)
            self.copy_out.wait_event(done)
            new_xyz.record_stream(self.copy_out)
            new_points.record_stream(self.copy_out)
            with torch.cuda.stream(self.copy_out):
                out_xyz_host[lo:hi].copy_(new_xyz, non_blocking=True)
                out_points_host[lo:hi].copy_(new_points, non_blocking=True)
        pn2.set_fps_mode(saved_mode)
        pn2.set_sa_engine(saved_engine)
        main.wait_stream(self.copy_out)
        main.wait_stream(self.copy_in)
        for s in self.streams:
            main.wait_stream(s)

    @torch.no_grad()
    def submit(self, host_feats: torch.Tensor, out_xyz_host: torch.Tensor, out_points_host: torch.Tensor) -> torch.cuda.Event:
        """Queue one whole batch: H2D into the free one of two device buffers (copy stream), the module over the full batch (compute
        stream) once it has landed, D2H of the results (third stream).  Nothing here waits for the previous batch except the reuse of
        a device buffer (two batches back) and the order of the result copies, so consecutive calls overlap copy and compute across
        batches.  Returns the event that marks this batch's results complete in the host buffers; the caller must not reuse
        ``host_feats`` before the copy has been consumed (``drain()`` or the event of the NEXT submit's results is enough)."""
        if self._ring is None or self._ring[0].shape != host_feats.shape:
            self._ring = [torch.empty(host_feats.shape, dtype=host_feats.dtype, device="cuda") for _ in range(2)]
            self._ring_free, self._submitted = [None, None], 0
        if self._submitted == 0:                                  # first batch after idle: order behind whatever the caller queued
            main = torch.cuda.current_stream()
            self.copy_in.wait_stream(main)
            self.streams[0].wait_stream(main)
            self.copy_out.wait_stream(main)
        slot = self._submitted % 2
        self._submitted += 1
        dev = self._ring[slot]
        if self._ring_free[slot] is not None:
            self.copy_in.wait_event(self._ring_free[slot])        # the batch two back has been read
        with torch.cuda.stream(self.copy_in):
            dev.copy_(host_feats, non_blocking=True)
            landed = torch.cuda.Event()
            landed.record(self.copy_in)
        s = self.streams[0]
        s.wait_event(landed)
        saved_mode, saved_engine = pn2._fps_mode, pn2._sa_engine
        if self.sa_engine is not None:
            pn2.set_sa_engine(self.sa_engine)
        pn2.set_fps_mode(self.fps_mode if self.fps_mode is not None else 0)
        with torch.cuda.stream(s):
            new_xyz, new_points = self.module(dev[:, :3].contiguous(), dev)
            if not new_xyz.is_contiguous():
                new_xyz = pn2.transpose_last2(new_xyz.permute(0, 2, 1))
            done = torch.cuda.Event()
            done.record(s)
        pn2.set_fps_mode(saved_mode)
        pn2.set_sa_engine(saved_engine)
        self._ring_free[slot] = done
        self.copy_out.wait_event(done)
        new_xyz.record_stream(self.copy_out)
        new_points.record_stream(self.copy_out)
        with torch.cuda.stream(self.copy_out):
            out_xyz_host.copy_(new_xyz, non_blocking=True)
            out_points_host.copy_(new_points, non_blocking=True)
            fin = torch.cuda.Event()
            fin.record(self.copy_out)
        self._last = fin
        return fin

    def drain(self) -> None:
        """Make the current stream wait for every submitted batch (results in their host buffers); the next submit starts a new run."""
        main = torch.cuda.current_stream()
        main.wait_stream(self.copy_in)
        main.wait_stream(self.streams[0])
        main.wait_stream(self.copy_out)
        self._submitted, self._ring_free = 0, [None, None]
