"""Restarting single rows of a stream (stream.restart) on the device: every session a row serves gives bit for bit what a
new batch_size=1 stream gives on the same chunks (and, in fp32, what one whole-clip call gives), the other rows are not
touched, graphs keep replaying, and the K/V cache follows the longest live clip.
Run on the H100 box:  python -m pytest tests -m gpu"""
import contextlib

import pytest
import torch

from oracle import weights as W
from tests.test_stream_gpu import _model
from tests.util import README_LAYERS, build_product

pytestmark = pytest.mark.gpu

CONFIGS = ["mini", "mini_gateloop", "mini_cond", "mini_fsq", "mini_mc", "mini_noff"]
PUSHES = 10
# rows restarted before push p: one restart after the first push, two rows in one push, rows restarting several times,
# restarts after the graphed stream's capture; row 0 is never restarted
RESTARTS = {1: [1], 3: [1, 2], 5: [2], 7: [1], 9: [2]}
README_KW = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)


def _sessions(restarts, B, P):
    """Per row, the [first push, end push) ranges of its sessions."""
    out = []
    for r in range(B):
        starts = [0] + [p for p in sorted(restarts) if r in restarts[p]]
        out.append(list(zip(starts, starts[1:] + [P])))
    return out


class _Schedule:
    """The chunks of B rows over P pushes, each row a sequence of sessions, and the cond of every session."""

    def __init__(self, model, side, B, P, restarts, seed, ff=True):
        self.model, self.side, self.B, self.P, self.restarts, self.ff = model, side, B, P, restarts, ff
        tdf = model.time_downsample_factor
        self.tp = tdf - 1 if self.ff else 0
        g = torch.Generator().manual_seed(seed)
        if side == "enc":
            self.sizes = [1 if self.ff else tdf] + [tdf] * (P - 1)
            self.sizes[min(5, P - 1)] = 2 * tdf                  # one push of 2 tdf frames
            self.x = W.synth_video(B, model.channels, sum(self.sizes), model.image_size, seed=seed).cuda()
        else:
            self.sizes = [1] * P
            q = model.quantizers
            shape = (B, P, model.fmap_size, model.fmap_size) + ((q.num_codebooks,) if q.num_codebooks > 1 else ())
            self.x = torch.randint(0, q.codebook_size, shape, generator=g).cuda()
        self.t0 = [sum(self.sizes[:p]) for p in range(P + 1)]
        self.conds = None
        if model.has_cond:      # the cond of each row at push 0, then of every restarted row
            self.conds = {0: torch.randn(B, model.dim_cond, generator=g).cuda()}
            for p, rows in restarts.items():
                self.conds[p] = torch.randn(len(rows), model.dim_cond, generator=g).cuda()

    def chunk(self, p):
        d = 2 if self.side == "enc" else 1
        return self.x.narrow(d, self.t0[p], self.sizes[p])

    def stream(self, B):
        kw = dict(batch_size=B, video_contains_first_frame=self.ff)
        if self.conds is not None:
            kw["cond"] = self.conds[0][:B]
        make = self.model.tokenize_stream if self.side == "enc" else self.model.decode_stream
        return make(**kw)

    def run(self, restarts=None, graphs=False, after=None):
        """The outputs of every push of one B-row stream, restarting rows as `restarts` says (default: the schedule's);
        after(p, stream) is called after push p."""
        restarts = self.restarts if restarts is None else restarts
        self.model.cuda_graphs = graphs
        try:
            s = self.stream(self.B)
            outs = []
            for p in range(self.P):
                if p in restarts:
                    s.restart(restarts[p], cond=None if self.conds is None else self.conds[p])
                outs.append(s.push(self.chunk(p)))
                if after is not None:
                    after(p, s)
        finally:
            self.model.cuda_graphs = False
        return outs

    def session_chunks(self, r, a, b):
        """The chunks of row r's session over pushes [a, b) as a new stream takes them: without the time padding that
        leads a restarted row's first encoder chunk."""
        chunks = [self.chunk(p)[r:r + 1] for p in range(a, b)]
        if a > 0 and self.side == "enc":
            chunks[0] = chunks[0][:, :, self.tp:]
        return chunks

    def session_cond(self, r, a):
        if self.conds is None:
            return None
        if a == 0:
            return self.conds[0][r:r + 1]
        return self.conds[a][self.restarts[a].index(r)][None]

    def session_out(self, outs, r, a, b):
        """Row r's outputs over its session [a, b), concatenated, less the padding frames the decoder returns in the
        session's first push."""
        d = 1 if self.side == "enc" else 2
        parts = [o[r:r + 1] for o in outs[a:b]]
        if a > 0 and self.side == "dec":
            parts[0] = parts[0][:, :, self.tp:]
        return torch.cat(parts, dim=d)

    def fresh(self, r, a, b):
        """What a new batch_size=1 stream gives on row r's session [a, b)."""
        kw = dict(batch_size=1, video_contains_first_frame=self.ff, cond=self.session_cond(r, a))
        s = (self.model.tokenize_stream if self.side == "enc" else self.model.decode_stream)(**kw)
        d = 1 if self.side == "enc" else 2
        return torch.cat([s.push(c) for c in self.session_chunks(r, a, b)], dim=d)

    def one_shot(self, r, a, b):
        """One whole-clip call on row r's session [a, b)."""
        m, cond = self.model, self.session_cond(r, a)
        clip = torch.cat(self.session_chunks(r, a, b), dim=2 if self.side == "enc" else 1)
        if self.side == "enc":
            return m(clip, cond=cond, return_codes=True, video_contains_first_frame=self.ff)
        return m.decode_from_code_indices(clip, cond=cond, video_contains_first_frame=self.ff)


def _schedule(name, dtype, side, B=3, P=PUSHES, restarts=RESTARTS, seed=31):
    g, model = _model(name, dtype)
    return _Schedule(model, side, B, P, restarts, seed, ff=name != "mini_noff")


def _check_sessions(sch, outs, one_shot=False):
    """Checks every session of `outs` (sch.run()) against a new stream; returns the number of sessions."""
    n = 0
    for r, sessions in enumerate(_sessions(sch.restarts, sch.B, sch.P)):
        for a, b in sessions:
            got = sch.session_out(outs, r, a, b)
            want = sch.fresh(r, a, b)
            assert got.dtype == want.dtype and torch.equal(got, want), (r, a, b, (got.float() - want.float()).abs().max())
            if one_shot:
                assert torch.equal(got, sch.one_shot(r, a, b)), (r, a, b)
            n += 1
    return n


@contextlib.contextmanager
def _tf32():
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev


@pytest.mark.parametrize("side", ["enc", "dec"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", CONFIGS)
def test_restarted_sessions_equal_new_streams(name, dtype, side):
    """Each session equals a new batch_size=1 stream on its chunks, and in fp32 one whole-clip call on its clip."""
    sch = _schedule(name, dtype, side)
    assert _check_sessions(sch, sch.run(), one_shot=dtype == torch.float32) == 9


@pytest.mark.parametrize("side", ["enc", "dec"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", CONFIGS)
def test_rows_never_restarted_are_untouched(name, dtype, side):
    sch = _schedule(name, dtype, side)
    outs, plain = sch.run(), sch.run(restarts={})
    for o, q in zip(outs, plain):
        assert torch.equal(o[:1], q[:1])


@pytest.mark.parametrize("side", ["enc", "dec"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", CONFIGS)
def test_graphed_restarts_replay(name, dtype, side):
    """With cuda_graphs the outputs are those of the eager stream, and the restarts after the capture (pushes 7 and 9)
    capture nothing new."""
    sch = _schedule(name, dtype, side)
    seen = {}
    graphed = sch.run(graphs=True, after=lambda p, s: seen.__setitem__(p, s.captures))
    eager = sch.run()
    assert all(torch.equal(a, b) for a, b in zip(graphed, eager))
    assert seen[6] >= 1 and seen[PUSHES - 1] == seen[6], seen


@pytest.mark.parametrize("graphs", [False, True])
def test_kv_cache_follows_the_longest_live_clip(graphs):
    """B = 4, 64 one-frame decoder pushes, each row restarted every 8 pushes, the rows' first restarts staggered: no
    session is longer than 8 latent frames, so the K/V cache never holds more than one growth step (16 frames); without
    dropping the frames of ended sessions it would reach 64.  Every session still equals a new stream."""
    P = 64
    restarts = {}
    for r in range(4):
        for p in range(2 * r + 1, P, 8):
            restarts.setdefault(p, []).append(r)
    sch = _schedule("mini", torch.bfloat16, "dec", B=4, P=P, restarts=restarts)
    step = sch.model.engine.KV_CACHE_STEP
    caps = []
    outs = sch.run(graphs=graphs, after=lambda p, s: caps.append(max(s.state.kv_capacities())))
    assert max(caps) == step == 16, caps
    assert _check_sessions(sch, outs) == 4 + sum(len(v) for v in restarts.values())


@pytest.mark.parametrize("side", ["enc", "dec"])
@pytest.mark.parametrize("precision", ["fp16", "tf32"])
def test_restarted_sessions_other_precisions(precision, side):
    dtype = torch.float16 if precision == "fp16" else torch.float32
    with _tf32() if precision == "tf32" else contextlib.nullcontext():
        sch = _schedule("mini", dtype, side)
        assert sch.stream(1).tf32 == (precision == "tf32")
        assert _check_sessions(sch, sch.run()) == 9


@pytest.mark.parametrize("side", ["enc", "dec"])
def test_readme_config_restarts_with_graphs(side):
    """README config, bf16, B = 4, graphs on: every row's sessions equal batch_size=1 streams."""
    torch.manual_seed(0)
    model = build_product(README_KW, 3).cuda().to(torch.bfloat16)
    restarts = {1: [1], 3: [1, 2], 5: [3], 7: [0, 2]}
    sch = _Schedule(model, side, 4, 9, restarts, seed=41)
    outs = sch.run(graphs=True)
    assert _check_sessions(sch, outs) == 10
    assert model.engine.fused_ru_calls > 0 and model.engine.slab_calls > 0
