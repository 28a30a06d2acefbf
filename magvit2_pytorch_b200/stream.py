"""Streaming tokenize and decode: a clip fed in chunks gives exactly the codes and frames of one whole-clip call.

The tokenizer is causal in time end to end (causal convs, TimeDownsample2x's window [2j-2, 2j], pointwise TimeUpsample2x,
right-aligned causal time attention with TokenShift, the gateloop forward scan), so chunk k's outputs depend only on frames up
to its own.  A stream carries what the next chunk needs from the earlier ones (engine.StreamState): per causal conv its last
k_t - 1 input frames, per token shift the previous frame, per time attention the qkv rows of every earlier frame, per
gateloop the fp32 scan state.  The kernels read that state in place (DESIGN.md 3.7).

    enc = tok.tokenize_stream(batch_size=B)
    codes = torch.cat([enc.push(chunk) for chunk in chunks], dim=1)      # == tok.tokenize(video)
    dec = tok.decode_stream(batch_size=B)
    video = torch.cat([dec.push(c) for c in codes.split(1, dim=1)], dim=2)   # == tok.decode_from_code_indices(codes)

With tok.cuda_graphs set, a stream replays its pushes as CUDA graphs (PushPlan) once it has seen a push of the same shape.

The rows of a stream are independent clips, and restart() starts single rows over, so one batched stream serves sessions
that begin and end at different times:

    dec.restart([2], cond=new_cond_row)      # row 2 starts a new clip at the next push
"""
from __future__ import annotations

import contextlib

import torch

from .engine import StreamState, tf32_matmul_enabled


def check_stream_model(model):
    """Construction-time checks shared by both streams (no device needed)."""
    for name in ("conv_in", "conv_out"):
        mode = getattr(model, name).pad_mode
        if mode != "constant":
            raise NotImplementedError(
                f"streaming needs pad_mode='constant' ({name} has '{mode}'): the other modes pad with the whole clip's "
                "leading frames, and only when the clip is longer than the padding, which a stream cannot know")


def encoder_chunk_frames(n: int, tdf: int, first_push: bool, first_frame: bool) -> int:
    """Latent frames an encoder push of n frames yields; ValueError names the chunk rule when n breaks it."""
    if first_push and first_frame:
        if n < 1 or (n - 1) % tdf:
            raise ValueError(f"the first push of a stream with a first frame takes 1 + k * {tdf} frames (k >= 0), got {n}")
        return (n - 1) // tdf + 1
    if n < tdf or n % tdf:
        what = "every later push" if first_frame else "every push of a stream without a first frame"
        raise ValueError(f"{what} takes k * {tdf} frames (k >= 1, the time downsample factor {tdf}), got {n}")
    return n // tdf


def decoder_chunk_frames(n: int, tdf: int, first_push: bool, first_frame: bool) -> int:
    """Frames a decoder push of n latent frames yields; ValueError when n < 1."""
    if n < 1:
        raise ValueError(f"a decoder push takes at least one latent frame, got {n}")
    return tdf * n - (tdf - 1 if first_push and first_frame else 0)


def restart_rows(rows, batch_size: int) -> list:
    """The row indices of a restart (a sequence of ints or a 1-D integer tensor) as a list; ValueError unless they are
    distinct and in [0, batch_size)."""
    if isinstance(rows, torch.Tensor):
        if rows.ndim != 1 or rows.dtype.is_floating_point or rows.dtype.is_complex or rows.dtype == torch.bool:
            raise ValueError(f"rows must be a 1-D integer tensor, got {rows.dtype} {tuple(rows.shape)}")
        rows = rows.tolist()
    else:
        rows = list(rows)
        if any(isinstance(r, bool) or not isinstance(r, int) for r in rows):
            raise ValueError(f"rows must be integers, got {rows}")
    if any(r < 0 or r >= batch_size for r in rows):
        raise ValueError(f"rows must lie in [0, {batch_size}), got {rows}")
    if len(set(rows)) != len(rows):
        raise ValueError(f"rows must be distinct, got {rows}")
    return rows


class PushPlan:
    """One push captured as CUDA graph segments, split where the push runs a host step (Engine.host_step: the streamed
    time attention, whose launch arguments change with every push).  A replay runs segment 0, host step 0, segment 1, ...
    on the current stream; the host steps read the stream's state as it is at that push.  All segments allocate from one
    private memory pool, so a segment may read what an earlier one wrote."""

    def __init__(self, eng, fn, x):
        """Captures fn(x), the push of input x (static copy: `x`), running each segment once as soon as it is captured so
        that the host step after it reads real values; the push's state update takes effect as in an eager push."""
        self.x = x.clone()
        self._eng = eng
        self._pool = torch.cuda.graph_pool_handle()
        self.graphs, self.launches, self.steps = [], [], []
        self._capture = None
        eng.host_step = self._split
        try:
            self._begin()
            self.out = fn(self.x)
            self._end()
        except BaseException:
            if self._capture is not None:
                self._capture.__exit__(None, None, None)
            raise
        finally:
            eng.host_step = None

    def _begin(self):
        g = torch.cuda.CUDAGraph()
        self._capture = torch.cuda.graph(g, pool=self._pool)
        self._capture.__enter__()
        self.graphs.append(g)
        self.launches.append(self._eng.launches)

    def _end(self):
        capture, self._capture = self._capture, None
        capture.__exit__(None, None, None)
        self.launches[-1] = self._eng.launches - self.launches[-1]
        self.graphs[-1].replay()

    def _split(self, step):
        self._end()
        out = step()
        self.steps.append(step)
        self._begin()
        return out

    def replay(self, x):
        """The push of input x -> its output (the plan's static output tensor)."""
        self.x.copy_(x, non_blocking=True)
        for i, (g, n) in enumerate(zip(self.graphs, self.launches)):
            if i:
                self.steps[i - 1]()
            g.replay()
            self._eng.launches += n
        return self.out


class _Stream:
    def __init__(self, model, batch_size, cond, video_contains_first_frame):
        check_stream_model(model)
        if int(batch_size) < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        self.model = model
        self.batch_size = int(batch_size)
        self.first_frame = bool(video_contains_first_frame)
        # the stream's own copy, in fp32 as the cond stems read it: restart() writes rows of it in place, so captured
        # pushes keep reading it
        cond = model._check_cond(cond, self.batch_size)
        self.cond = None if cond is None else cond.detach().to(torch.float32, copy=True).contiguous()
        self._restarted = set()      # rows restarted since the last push
        self.state = StreamState()
        # an fp32 model's precision is read from torch's TF32 switch once, here: every push runs in it, so the pushes still
        # give the outputs of one whole-clip call in that precision bit for bit
        self.tf32 = model.dtype == torch.float32 and tf32_matmul_enabled()
        self.pushes = 0
        self._sig_id = None
        self._plans = {}             # push signature -> "warm" | PushPlan (model.cuda_graphs)
        self.captures = 0            # PushPlans captured

    @contextlib.contextmanager
    def _engine(self):
        """The model's engine in this stream's precision for one push, eval mode, checked against the parameter packs this
        stream started with."""
        self.model.eval()
        eng = self.model.engine
        if self._sig_id is None:
            self._sig_id = eng._sig_id
        elif eng._sig_id != self._sig_id:
            raise RuntimeError("the tokenizer's parameters changed while this stream was open: its carried state belongs "
                               "to the old ones; start a new stream")
        prev, eng.tf32 = eng.tf32, self.tf32
        try:
            if self.tf32:
                eng.prepare()         # adds the TF32 packs on the first such push
            yield eng
        finally:
            eng.tf32 = prev

    def _run(self, eng, fn, x, first, sff_rest):
        """fn(x), the push of input x.  With model.cuda_graphs set it goes through this stream's PushPlans, with the rule
        VideoTokenizer._graph_call follows: the first push of a signature runs eagerly, the second is captured, later ones
        replay.  The signature is what the push's launches depend on besides the K/V cache length its host steps read: the
        input's shape and dtype, the first-push flags and every conv history's frame count.  A replay does not update the
        counts, so only pushes that leave them unchanged are captured; the others (the first few, while the histories
        fill up) run eagerly, and their signatures do not recur."""
        if not self.model.cuda_graphs:
            return fn(x)
        counts = self.state.history_counts()
        key = (tuple(x.shape), x.dtype, first, sff_rest, counts)
        plan = self._plans.get(key)
        if plan is None:
            out = fn(x)
            if self.state.history_counts() == counts:
                self._plans[key] = "warm"
            return out
        if plan == "warm":
            plan = self._plans[key] = PushPlan(eng, fn, x)
            self.captures += 1
            out = plan.out
        else:
            out = plan.replay(x)
        return out.clone()

    def restart(self, rows, cond=None):
        """Rows `rows` (distinct indices, a list or a 1-D integer tensor) start new clips at the next push; the other rows
        carry on.  cond: (len(rows), dim_cond), the new clips' cond, required exactly when the model has cond layers.

        From the next push on, a restarted row computes what a new batch_size=1 stream computes from its new clip's chunks,
        and the other rows what they would without the restart.  Pushes keep their chunk rule: with a first frame, in a
        restarted row's first push the first tdf - 1 frames of an encoder chunk are the clip's time padding (their values
        are ignored, zeros are used) and the first tdf - 1 frames a decoder push returns are the padding that the
        whole-clip decode drops.  Before the stream's first push a restart only replaces cond."""
        m = self.model
        if m.separate_first_frame_encoding and self.first_frame:
            raise NotImplementedError(
                "restart is not supported with separate_first_frame_encoding and a first frame: the first frame takes the "
                "2-D conv for the whole push")
        rows = restart_rows(rows, self.batch_size)
        if m.has_cond:
            if not isinstance(cond, torch.Tensor) or tuple(cond.shape) != (len(rows), m.dim_cond) \
                    or not cond.dtype.is_floating_point:
                got = f"{cond.dtype} {tuple(cond.shape)}" if isinstance(cond, torch.Tensor) else repr(cond)
                raise ValueError(f"cond must be a float ({len(rows)}, {m.dim_cond}) tensor, got {got}")
            if cond.device != m.device:
                raise ValueError(f"cond is on {cond.device} but the tokenizer is on {m.device}")
            if rows:
                self.cond[rows] = cond.detach().to(self.cond.dtype)
        if self.pushes and rows:
            with torch.cuda.device(m.device):
                self.state.restart_rows(rows)
            self._restarted.update(rows)

    def _check_batch(self, t, what):
        if t.shape[0] != self.batch_size:
            raise ValueError(f"{what} has batch {t.shape[0]}, the stream was built for batch_size={self.batch_size}")
        self.model._check_on_device(t, what)


class TokenizeStream(_Stream):
    """Encoder + quantiser of a clip fed in chunks; see push()."""

    @torch.no_grad()
    def push(self, chunk: torch.Tensor) -> torch.Tensor:
        """chunk (B, C, n, H, W) float / bf16 / uint8 frames -> codes (B, n', H', W'[, num_codebooks]) of those frames:
        n' = n // tdf, plus 1 on the first push of a stream with a first frame (which takes 1 + k * tdf frames).  With a
        first frame, the first tdf - 1 frames of a row's chunk in its first push after a restart are read as zeros."""
        m = self.model
        if chunk.ndim != 5 or chunk.shape[1] != m.channels or tuple(chunk.shape[-2:]) != (m.image_size, m.image_size):
            raise ValueError(f"chunk must be (B, {m.channels}, n, {m.image_size}, {m.image_size}), got {tuple(chunk.shape)}")
        self._check_batch(chunk, "chunk")
        first = self.pushes == 0
        encoder_chunk_frames(chunk.shape[2], m.time_downsample_factor, first, self.first_frame)
        ff, sff_rest = self.first_frame and first, self.first_frame and not first and m.separate_first_frame_encoding
        with torch.cuda.device(m.device), self._engine() as eng:
            def fn(v):
                return eng.quantize_cl(eng.encode_cl(v, ff, self.cond, ss=self.state, sff_rest=sff_rest),
                                       want_quantized=False)[1]
            x = chunk.contiguous()
            if self._restarted and self.first_frame:
                # the new clips' time padding, which the whole-clip call prepends as zero frames, on a copy of the chunk
                x = x.clone()
                for r in self._restarted:
                    x[r, :, :m.time_padding].zero_()
            codes = self._run(eng, fn, x, first, sff_rest)
        self.pushes += 1
        self._restarted.clear()
        return codes


class DecodeStream(_Stream):
    """Decoder of latent codes fed in chunks; see push()."""

    @torch.no_grad()
    def push(self, codes: torch.Tensor) -> torch.Tensor:
        """codes (B, n', H', W'[, num_codebooks]) int64 / int32 -> frames (B, C, tdf * n', H, W) in the model dtype, less the
        time_padding frames on the first push of a stream with a first frame.  With a first frame, the first tdf - 1
        frames of a row in its first push after a restart are that padding, for the caller to drop."""
        m = self.model
        nc = m.quantizers.num_codebooks
        if codes.dtype not in (torch.long, torch.int32) or codes.ndim != (4 if nc == 1 else 5) or \
                (nc > 1 and codes.shape[-1] != nc):
            raise ValueError(f"codes must be int64 / int32 (B, n, H, W{'' if nc == 1 else ', num_codebooks'}), "
                             f"got {codes.dtype} {tuple(codes.shape)}")
        self._check_batch(codes, "codes")
        first = self.pushes == 0
        decoder_chunk_frames(codes.shape[1], m.time_downsample_factor, first, self.first_frame)
        ff, sff_rest = self.first_frame and first, self.first_frame and not first and m.separate_first_frame_encoding
        with torch.cuda.device(m.device), self._engine() as eng:
            def fn(c):
                return eng.decode_cl(eng.codes_to_quantized_cl(c), ff, self.cond, ss=self.state, sff_rest=sff_rest)
            out = self._run(eng, fn, codes.contiguous(), first, sff_rest)
        self.pushes += 1
        self._restarted.clear()
        return out
