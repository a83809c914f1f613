"""EncoderRunner: the sync-free, CUDA-graph way to call the encoder half for a fixed batch geometry.

The reference forces ~40 host synchronisations and ~1000 tiny launches per encoder forward (SURVEY.md 3a);
on an H100 the algorithmic time of the path is ~0.1-1 ms, so launch latency would dominate.  The runner builds
the ``EncoderPlan`` once, captures ``SalienceTransformer.forward_encoder`` into one CUDA graph over static
device buffers and replays it; ``run_host`` adds the pinned-host <-> device copies on the same stream."""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import cabi
from .salience_transformer import SalienceTransformer


class HostPipeline:
    """Double-buffered host -> device -> host streaming over two EncoderRunners of the same geometry.

    H2D copies (copy stream), the encoder graph (compute stream) and the D2H copy of the memory (second copy
    stream) of consecutive batches overlap; a batch's buffers are reused only after its D2H has finished.
    PCIe is full duplex, so the steady-state step time is max(compute, H2D, D2H) instead of their sum."""

    def __init__(self, model: SalienceTransformer, feats, masks, pos, depth: int = 2, **kw):
        self.lanes = [EncoderRunner(model, feats, masks, pos, **kw) for _ in range(depth)]
        dev = self.lanes[0].dev
        self.h2d = torch.cuda.Stream(device=dev)
        self.d2h = torch.cuda.Stream(device=dev)
        self.done = [None] * depth       # event: D2H of the lane's previous batch finished (its output buffers are free)
        self.computed = [None] * depth   # event: forward of the lane's previous batch finished (its input buffers are free)
        self.host_out = [torch.empty(self.lanes[0].memory.shape, dtype=torch.float32, pin_memory=True)
                         for _ in range(depth)]
        self.h2d_bytes = self.d2h_bytes = 0

    def run(self, batches, on_output=None):
        """batches: iterable of (feats_host, pos_host) pinned-memory level lists (pos_host None / empty when the runners
        derive the position embedding from the masks on the device).  Returns the number processed;
        ``on_output(i, host_memory)`` (optional) is called, in batch order, once batch i's output is in host memory.
        ``host_memory`` is the lane's pinned buffer: consume or copy it before returning -- a later batch overwrites it."""
        n = 0
        for i, (feats_h, pos_h) in enumerate(batches):
            k = i % len(self.lanes)
            lane = self.lanes[k]
            if self.computed[k] is not None:
                self.h2d.wait_event(self.computed[k])      # the lane's INPUT buffers are free once its forward is done
            if self.done[k] is not None and on_output is not None:
                self.done[k].synchronize()
                on_output(i - len(self.lanes), self.host_out[k])
            with torch.cuda.stream(self.h2d):
                for dst, src in zip(lane.feats + lane.pos, list(feats_h) + list(pos_h or [])):
                    dst.copy_(src, non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(self.h2d)
            lane.stream.wait_event(ready)
            if self.done[k] is not None:
                lane.stream.wait_event(self.done[k])       # the lane's OUTPUT buffer was copied out
            mem = lane.step()
            computed = torch.cuda.Event()
            computed.record(lane.stream)
            self.computed[k] = computed
            self.d2h.wait_event(computed)
            with torch.cuda.stream(self.d2h):
                self.host_out[k].copy_(mem, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self.d2h)
            self.done[k] = ev
            n += 1
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in self.lanes[0].feats + self.lanes[0].pos)
        self.d2h_bytes = self.host_out[0].numel() * 4
        depth = len(self.lanes)
        for i in range(max(0, n - depth), n):   # drain: the last `depth` batches, in batch order
            k = i % depth
            self.done[k].synchronize()
            if on_output is not None:
                on_output(i, self.host_out[k])
        return n


class FreshMaskPipeline:
    """Host -> device -> host streaming for batches whose PADDING MASKS DIFFER from batch to batch (the detector's normal input:
    every batch is padded to its own largest image).  Nothing derived from the masks can be reused, and the top-k sizes of the
    plan are host integers, so a captured graph cannot be replayed: each batch runs ``make_plan`` (two launches + one small
    device -> host copy) and an EAGER ``forward_encoder``.  What can still overlap does: the H2D copy of batch i+1 (copy
    stream), the plan of batch i+1 (its own stream, so the host round trip waits for the mask copy and two small kernels only, not
    for the forwards in flight), the forward of batch i (lane stream) and the D2H copy of batch i-1 (second copy stream).  The host
    issues ~120 launches per forward, which is what bounds the rate once the copies are hidden (tools/profile_eager_cpu.py).

    All batches must have the padded geometry (level shapes, batch size) of the ``feats`` / ``masks`` given here."""

    def __init__(self, model: SalienceTransformer, feats, masks, depth: int = 3, use_order: bool = True):
        self.model = model.eval()
        self.dev = feats[0].device
        self.use_order = use_order
        self.depth = depth
        self.feats = [[torch.empty_like(f) for f in feats] for _ in range(depth)]
        self.masks = [[torch.empty_like(m) for m in masks] for _ in range(depth)]
        self.streams = [torch.cuda.Stream(device=self.dev) for _ in range(depth)]
        self.h2d = torch.cuda.Stream(device=self.dev)
        self.d2h = torch.cuda.Stream(device=self.dev)
        self.plan_stream = torch.cuda.Stream(device=self.dev, priority=-1)
        self.done = [None] * depth
        self.computed = [None] * depth
        self.keep = [None] * depth       # the lane's plan / output tensors stay referenced until its buffers are reused
        self.host_out = None
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in list(feats) + list(masks))
        self.d2h_bytes = 0

    def run(self, batches, on_output=None):
        """batches: iterable of (feats_host, masks_host) pinned-memory level lists.  ``on_output(i, host_memory)`` as in
        ``HostPipeline.run``.  Returns the number processed."""
        n = 0
        for i, (feats_h, masks_h) in enumerate(batches):
            k = i % self.depth
            if self.computed[k] is not None:
                self.h2d.wait_event(self.computed[k])
            if self.done[k] is not None:
                self.done[k].synchronize()       # also bounds how far the host runs ahead of the device
                if on_output is not None:
                    on_output(i - self.depth, self.host_out[k])
            with torch.cuda.stream(self.h2d):
                for dst, src in zip(self.masks[k], masks_h):   # masks first: the plan needs only them
                    dst.copy_(src, non_blocking=True)
                masks_ready = torch.cuda.Event()
                masks_ready.record(self.h2d)
                for dst, src in zip(self.feats[k], feats_h):
                    dst.copy_(src, non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(self.h2d)
            self.plan_stream.wait_event(masks_ready)
            with torch.cuda.stream(self.plan_stream), torch.no_grad():
                plan = self.model.make_plan(self.masks[k])   # host round trip: waits for the mask copy and the plan kernels only
                planned = torch.cuda.Event()
                planned.record(self.plan_stream)
            s = self.streams[k]
            s.wait_event(planned)
            s.wait_event(ready)
            with torch.cuda.stream(s), torch.no_grad():
                mem, _ = self.model.forward_encoder(self.feats[k], self.masks[k], None, plan=plan, use_order=self.use_order)
                computed = torch.cuda.Event()
                computed.record(s)
            self.computed[k] = computed
            if self.host_out is None:
                self.host_out = [torch.empty(mem.shape, dtype=torch.float32, pin_memory=True) for _ in range(self.depth)]
                self.d2h_bytes = mem.numel() * 4
            self.d2h.wait_event(computed)
            with torch.cuda.stream(self.d2h):
                self.host_out[k].copy_(mem, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self.d2h)
            self.done[k] = ev
            self.keep[k] = (plan, mem)
            n += 1
        for i in range(max(0, n - self.depth), n):
            k = i % self.depth
            self.done[k].synchronize()
            if on_output is not None:
                on_output(i, self.host_out[k])
        return n


class EncoderRunner:
    def __init__(self, model: SalienceTransformer, feats: Sequence[torch.Tensor], masks: Sequence[torch.Tensor],
                 pos: Sequence[torch.Tensor], use_graph: bool = True, use_order: bool = True, warmup: int = 2):
        self.model = model.eval()
        self.dev = feats[0].device
        self.feats = [f.clone() for f in feats]      # static device buffers (graph inputs)
        # pos None: the sine position embedding is derived from the masks on the device, once per plan, in token layout
        # (model.attach_position_embedding) -- nothing to copy per step
        self.pos = [p.clone() for p in pos] if pos is not None else []
        self.masks = [m.clone() for m in masks]
        self.use_order = use_order
        with torch.no_grad():
            self.plan = model.make_plan(self.masks)  # the single host round trip of this geometry
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_step = 0
        self.memory: Optional[torch.Tensor] = None
        self.stream = torch.cuda.Stream(device=self.dev)
        self._host_in: Optional[List[torch.Tensor]] = None
        self._host_out: Optional[torch.Tensor] = None
        s = self.stream
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(max(1, warmup)):          # also sizes cuBLAS workspaces before capture
                n0 = cabi.launch_count()
                self.memory, _ = self.model.forward_encoder(self.feats, self.masks, self.pos or None, plan=self.plan,
                                                            use_order=self.use_order)
                self.launches_per_step = cabi.launch_count() - n0
        s.synchronize()
        if use_graph:
            g = torch.cuda.CUDAGraph()
            with torch.no_grad(), torch.cuda.graph(g, stream=s):
                self.memory, _ = self.model.forward_encoder(self.feats, self.masks, self.pos or None, plan=self.plan,
                                                            use_order=self.use_order)
            self.graph = g
        torch.cuda.current_stream(self.dev).wait_stream(s)

    def step(self) -> torch.Tensor:
        """One encoder-half forward over the static device buffers, on ``self.stream``; returns ``memory``."""
        with torch.cuda.stream(self.stream), torch.no_grad():
            if self.graph is not None:
                self.graph.replay()
            else:
                self.memory, _ = self.model.forward_encoder(self.feats, self.masks, self.pos or None, plan=self.plan,
                                                            use_order=self.use_order)
        return self.memory

    # -- host I/O ------------------------------------------------------------------------------------------------
    def bind_host(self, feats_h: Sequence[torch.Tensor], pos_h: Optional[Sequence[torch.Tensor]] = None):
        """Pinned host staging for ``run_host`` (feature maps and -- unless derived on the device -- position embeddings)."""
        self._host_in = [t.pin_memory() if not t.is_pinned() else t for t in list(feats_h) + list(pos_h or [])]
        self._host_out = torch.empty(self.memory.shape, dtype=self.memory.dtype, pin_memory=True)
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in self._host_in)
        self.d2h_bytes = self._host_out.numel() * self._host_out.element_size()

    def run_host(self) -> torch.Tensor:
        """host (pinned) -> device copies, forward, device -> host copy of the encoder memory; all on one stream.
        Masks (and hence the plan) are fixed for the runner's geometry.  Asynchronous: synchronise ``self.stream``
        before reading the returned pinned buffer."""
        n = len(self.feats)
        with torch.cuda.stream(self.stream):
            for dst, src in zip(self.feats + self.pos, self._host_in):
                dst.copy_(src, non_blocking=True)
        mem = self.step()
        with torch.cuda.stream(self.stream):
            self._host_out.copy_(mem, non_blocking=True)
        return self._host_out
