"""Pinned-host-buffer front end of the tokenizer round trip.

A caller that keeps its videos and results in host memory (a data loader on one side, a token store on the other) pays
a host->device copy before and a device->host copy after every `tokenize` / `decode_from_code_indices` call of the
reference API (magvit2_pytorch.py M:1651-1654, M:1590-1617).  `HostRoundTrip` issues the three phases on three CUDA
streams with `depth` device staging slots, so the H2D copy of call i+1 and the D2H copy of call i-1 run under the
kernels of call i.  Nothing is computed differently: the kernels are the ones `VideoTokenizer.tokenize` /
`.decode_from_code_indices` launch, on the caller's current stream (or, with `lanes` > 1, on `lanes` compute streams so
that the kernels of consecutive calls overlap too: `StreamLanes`).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .engine import tf32_matmul_enabled


class StreamLanes:
    """`lanes` CUDA streams, each with its own CUDA-graph instances of the model's entry points (`VideoTokenizer._lane`).

    A step of this path is a chain of ~170 dependent launches: tensor-pipe-bound convolutions alternate with HBM-bound
    (gate / residual, norms, SE pooling) and latency-bound (SE gate MLP, small attention) kernels, and a persistent conv
    kernel occupies one CTA per SM.  Independent calls (different batches) issued on different lanes let the hardware
    fill the HBM- and latency-bound phases of one call with the tensor-bound phases of another.  Nothing is computed
    differently: every call replays the same kernels on the same data layout; only the stream differs.

    ``run(fn, *args)`` executes ``fn(*args)`` with the next lane's stream current and returns ``(result, event)``; the lane
    first waits for the caller's current stream (the inputs' producer).  The caller consumes the result on its own stream
    after ``stream.wait_event(event)`` (or after ``join()``)."""

    def __init__(self, model, lanes: int = 2):
        assert lanes >= 1
        self.model = model
        self.device = model.device
        if self.device.type != "cuda":
            raise RuntimeError("StreamLanes needs the tokenizer on a CUDA device")
        self.streams = [torch.cuda.Stream(self.device) for _ in range(lanes)]
        self.events = [torch.cuda.Event() for _ in range(lanes)]
        self.n = 0

    def next_lane(self) -> int:
        lane = self.n % len(self.streams)
        self.n += 1
        return lane

    def run_on(self, lane: int, fn, *args):
        s = self.streams[lane]
        # (re)pack the parameters, if they changed, on the CALLER's stream: every lane is ordered after it below, so no lane
        # can read packs that another lane's stream is still writing
        eng = self.model.engine
        if eng.dtype == torch.float32 and tf32_matmul_enabled():
            eng.prepare(tf32_packs=True)        # the TF32 packs the call will add
        s.wait_stream(torch.cuda.current_stream(self.device))
        prev = self.model._lane
        self.model._lane = lane
        try:
            with torch.cuda.stream(s):
                res = fn(*args)
                self.events[lane].record(s)
        finally:
            self.model._lane = prev
        return res, self.events[lane]

    def run(self, fn, *args):
        return self.run_on(self.next_lane(), fn, *args)

    def join(self) -> None:
        """Makes the caller's current stream wait for everything issued on the lanes so far."""
        cur = torch.cuda.current_stream(self.device)
        for s in self.streams:
            cur.wait_stream(s)


class _Slot:
    __slots__ = ("video", "codes", "recon", "h2d", "done", "d2h", "used")

    def __init__(self):
        self.video: Optional[torch.Tensor] = None
        self.codes = self.recon = None
        self.h2d = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.d2h = torch.cuda.Event()
        self.used = False


class HostRoundTrip:
    """``submit(video_host, out_codes_host, out_video_host)`` enqueues copy-in -> tokenize -> decode -> copy-out and
    returns a CUDA event that completes when both host outputs are written.  All host tensors must be pinned.  The
    caller's buffers of a submit may be reused once its event has completed (``wait(event)``) or after
    ``synchronize()``; at most `depth` submits are in flight on the device side."""

    def __init__(self, model, depth: int = 2, train_mode_forward: bool = False, lanes: int = 1):
        assert depth >= 1 and 1 <= lanes <= depth
        self.model = model
        # True: one ``model(video, return_codes=True, return_recon=True)`` call per submit (in ``model.train()`` this is the
        # path with the LFQ batch-entropy all-reduce, BASELINE configs[2]) instead of tokenize + decode_from_code_indices
        self.train_mode_forward = train_mode_forward
        self.device = model.device
        if self.device.type != "cuda":
            raise RuntimeError("HostRoundTrip needs the tokenizer on a CUDA device")
        self.s_in = torch.cuda.Stream(self.device)
        self.s_out = torch.cuda.Stream(self.device)
        self.slots: List[_Slot] = [_Slot() for _ in range(depth)]
        # lanes > 1: the kernels of slot i run on compute stream i % lanes (StreamLanes) instead of the caller's current
        # stream, so the kernels of up to `lanes` consecutive submits overlap on the device as well
        self.lanes = StreamLanes(model, lanes) if lanes > 1 else None
        self.n = 0

    def submit(self, video_host: torch.Tensor, out_codes_host: torch.Tensor, out_video_host: torch.Tensor) -> torch.cuda.Event:
        for t in (video_host, out_codes_host, out_video_host):
            if t.device.type != "cpu" or not t.is_pinned():
                raise ValueError("HostRoundTrip takes pinned host tensors")
        slot = self.slots[self.n % len(self.slots)]
        self.n += 1
        cur = torch.cuda.current_stream(self.device)
        if slot.video is None or slot.video.shape != video_host.shape or slot.video.dtype != video_host.dtype:
            if slot.used:
                slot.done.synchronize()
            slot.video = torch.empty(video_host.shape, dtype=video_host.dtype, device=self.device)
            # the block may have been freed on `cur` with kernels still queued there: order the first copy after them
            self.s_in.wait_stream(cur)
        if slot.used:
            self.s_in.wait_event(slot.done)          # the kernels that read this slot's staged input have finished
        with torch.cuda.stream(self.s_in):
            slot.video.copy_(video_host, non_blocking=True)
            slot.h2d.record(self.s_in)
        lane = ((self.n - 1) % len(self.slots)) % len(self.lanes.streams) if self.lanes is not None else 0
        sc = self.lanes.streams[lane] if self.lanes is not None else cur
        if sc is not cur:
            # parameter (re)packing, and the TF32 packs the calls may add, happen on `cur`, which every lane waits for
            eng = self.model.engine
            if eng.dtype == torch.float32 and tf32_matmul_enabled():
                eng.prepare(tf32_packs=True)
            sc.wait_stream(cur)                      # whatever the caller queued before this submit (weight updates, ...)
        sc.wait_event(slot.h2d)
        if slot.used:
            sc.wait_event(slot.d2h)                  # the slot's previous results have left the device
        prev_lane = self.model._lane
        self.model._lane = lane
        try:
            with torch.cuda.stream(sc):
                if self.train_mode_forward:
                    codes, recon = self.model(slot.video, return_codes=True, return_recon=True)
                else:
                    codes = self.model.tokenize(slot.video)
                    recon = self.model.decode_from_code_indices(codes)
                slot.done.record(sc)
        finally:
            self.model._lane = prev_lane
        slot.codes, slot.recon = codes, recon        # keep the device results alive until their D2H copy is done
        self.s_out.wait_event(slot.done)
        with torch.cuda.stream(self.s_out):
            out_codes_host.copy_(codes, non_blocking=True)
            out_video_host.copy_(recon, non_blocking=True)
            slot.d2h.record(self.s_out)
        slot.used = True
        return slot.d2h

    @staticmethod
    def wait(event: torch.cuda.Event) -> None:
        event.synchronize()

    def join(self) -> None:
        """Makes the caller's current stream wait for the device->host copies of every submit so far."""
        cur = torch.cuda.current_stream(self.device)
        for s in self.slots:
            if s.used:
                cur.wait_event(s.d2h)

    def synchronize(self) -> None:
        for s in self.slots:
            if s.used:
                s.d2h.synchronize()
