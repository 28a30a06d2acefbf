"""Streaming tokenize / decode with cuda_graphs on (stream.PushPlan): pushes after the warm-up replay captured CUDA graph
segments around the time attention's host steps, and give bit for bit what the same pushes give eagerly and what one
whole-clip call gives.  Run on the H100 box:  python -m pytest tests -m gpu"""
import pytest
import torch

from magvit2_pytorch_b200.stream import PushPlan
from oracle import weights as W
from tests.test_stream_gpu import CONFIGS, _model, _one_shot
from tests.util import README_LAYERS, build_product

pytestmark = pytest.mark.gpu

README_KW = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)


def _pushes(stream, x, sizes, dim_out):
    """The outputs of pushing chunks of `sizes` frames of x, concatenated: video (time dim 2) to a TokenizeStream, whose
    codes have time dim 1 (dim_out = 1), or codes to a DecodeStream (dim_out = 2)."""
    outs, t = [], 0
    for n in sizes:
        outs.append(stream.push(x.narrow(3 - dim_out, t, n)))
        t += n
    return torch.cat(outs, dim=dim_out)


class _Replays:
    """Counts PushPlan replays while active."""

    def __init__(self, monkeypatch):
        self.n = 0
        orig = PushPlan.replay

        def replay(plan, x):
            self.n += 1
            return orig(plan, x)
        monkeypatch.setattr(PushPlan, "replay", replay)


def _both(model, make, x, sizes, dim_out):
    """(graphs-off outputs, graphs-on outputs, the graphs-on stream) of the same pushes on two new streams."""
    model.cuda_graphs = False
    eager = _pushes(make(), x, sizes, dim_out)
    model.cuda_graphs = True
    s = make()
    graphed = _pushes(s, x, sizes, dim_out)
    model.cuda_graphs = False
    return eager, graphed, s


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", CONFIGS)
def test_graphed_stream_equals_eager_stream_and_one_shot(monkeypatch, name, dtype):
    """One latent frame per push: the histories fill in the first pushes, the next one warms up, the one after is
    captured and the rest replay.  8 latent frames keep the time attention within the short-sequence kernel's L <= 8 in
    bf16 (DESIGN.md 3.7); the tdf = 2 configs, which have no time attention, take 10, as conv_in's 6-frame history needs
    three 2-frame pushes to fill."""
    g, model = _model(name, dtype)
    ff = name != "mini_noff"
    tdf = model.time_downsample_factor
    n_lat = 10 if tdf == 2 else 8
    video = W.synth_video(2, 3, (1 + (n_lat - 1) * tdf) if ff else n_lat * tdf, model.image_size, seed=21).cuda()
    cond = g["cond"].cuda() if model.has_cond else None
    codes, recon = _one_shot(model, video, cond, ff)
    replays = _Replays(monkeypatch)
    kw = dict(batch_size=2, cond=cond, video_contains_first_frame=ff)

    sched = ([1] + [tdf] * (n_lat - 1)) if ff else [tdf] * n_lat
    eager, graphed, enc = _both(model, lambda: model.tokenize_stream(**kw), video, sched, 1)
    assert torch.equal(eager, codes) and torch.equal(graphed, codes)
    assert enc.captures == 1 and replays.n >= 3, (enc.captures, replays.n)

    replays.n = 0
    eager, graphed, dec = _both(model, lambda: model.decode_stream(**kw), codes, [1] * n_lat, 2)
    assert graphed.dtype == recon.dtype and torch.equal(eager, recon) and torch.equal(graphed, recon)
    assert dec.captures == 1 and replays.n >= 3, (dec.captures, replays.n)


def test_readme_decode_stream_across_cache_growths():
    """README config, bf16: 40 one-frame decoder pushes cross the short-sequence kernel's L = 8 limit and two K/V cache
    growths (16 -> 32 -> 48 frames), all in the host steps between replayed segments."""
    torch.manual_seed(0)
    model = build_product(README_KW, 3).cuda().to(torch.bfloat16)
    codes = torch.randint(0, 1024, (2, 40, 16, 16), device="cuda")
    eager, graphed, dec = _both(model, lambda: model.decode_stream(batch_size=2), codes, [1] * 40, 2)
    assert dec.captures == 1 and torch.equal(graphed, eager)


def test_interleaved_graphed_streams_and_one_shot_calls():
    """Two open streams of one model, with graphed one-shot calls between their pushes: each stream owns its state and
    its graphs."""
    g, model = _model("mini_gateloop", torch.float32)
    va = W.synth_video(2, 3, 25, 32, seed=1).cuda()
    vb = W.synth_video(2, 3, 25, 32, seed=2).cuda()
    ref_a, ref_b = model.tokenize(va), model.tokenize(vb)
    model.cuda_graphs = True
    ea, eb = model.tokenize_stream(batch_size=2), model.tokenize_stream(batch_size=2)
    outs_a, outs_b = [], []
    for t0 in [0] + list(range(1, 25, 4)):
        n = 1 if t0 == 0 else 4
        outs_a.append(ea.push(va[:, :, t0:t0 + n]))
        assert torch.equal(model.tokenize(vb), ref_b)          # a one-shot call between pushes
        outs_b.append(eb.push(vb[:, :, t0:t0 + n]))
    assert torch.equal(torch.cat(outs_a, 1), ref_a) and torch.equal(torch.cat(outs_b, 1), ref_b)
    assert ea.captures == eb.captures == 1


def test_captures_stay_bounded_and_replays_count_the_eager_launches():
    """Pushes of 1 and 2 latent frames in turn: one plan per size, captured once.  Each push adds to Engine.launches what
    the same push adds on a graphs-off stream.  Turning cuda_graphs off and on mid-stream keeps the outputs exact."""
    g, model = _model("mini", torch.bfloat16)
    eng = model.engine
    codes = torch.randint(0, 1024, (2, 24, 4, 4), device="cuda")
    sizes = [1, 2] * 8

    def run(graphs, toggle=False):
        dec = model.decode_stream(batch_size=2)
        outs, added, t = [], [], 0
        for i, n in enumerate(sizes):
            model.cuda_graphs = graphs and not (toggle and i in (10, 11))
            torch.cuda.synchronize()
            l0 = eng.launches
            outs.append(dec.push(codes[:, t:t + n]))
            torch.cuda.synchronize()
            added.append(eng.launches - l0)
            t += n
        model.cuda_graphs = False
        return torch.cat(outs, 2), added, dec

    eager, n_eager, _ = run(False)
    graphed, n_graphed, dec = run(True)
    assert torch.equal(graphed, eager) and n_graphed == n_eager, (n_graphed, n_eager)
    assert dec.captures == 2 and sum(isinstance(p, PushPlan) for p in dec._plans.values()) == 2
    toggled, _, dec = run(True, toggle=True)
    assert torch.equal(toggled, eager) and dec.captures == 2


def test_parameter_change_raises_with_graphs():
    g, model = _model("mini", torch.float32)
    model.cuda_graphs = True
    enc = model.tokenize_stream(batch_size=2)
    v = W.synth_video(2, 3, 25, 32, seed=1).cuda()
    enc.push(v[:, :, :1])
    for t in range(1, 21, 4):                                   # warm-up, capture and replays
        enc.push(v[:, :, t:t + 4])
    assert enc.captures == 1
    with torch.no_grad():
        model.conv_in.conv.weight.mul_(1.0)                     # an in-place edit: the packs are rebuilt
    with pytest.raises(RuntimeError, match="parameters changed"):
        enc.push(v[:, :, 21:25])


def test_graphed_decode_stream_memory_grows_with_the_kv_cache_only():
    """As tests/test_stream_gpu.py's eager test: with graphs, the peak allocation of one-frame pushes 8..64 grows by the
    time attention's K/V cache only; the captured plan's memory pool was allocated before push 8."""
    torch.manual_seed(0)
    model = build_product(README_KW, 3).cuda().to(torch.bfloat16)
    model.cuda_graphs = True
    codes = torch.randint(0, 1024, (1, 64, 16, 16), device="cuda")
    dec = model.decode_stream(batch_size=1)
    for i in range(8):
        dec.push(codes[:, i:i + 1])
    assert dec.captures == 1
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for i in range(8, 16):
        dec.push(codes[:, i:i + 1])
    peak8 = torch.cuda.max_memory_allocated()
    for i in range(16, 64):
        dec.push(codes[:, i:i + 1])
    peak64 = torch.cuda.max_memory_allocated()
    at = model.decoder_layers[0][0].fn.fn
    kv = 16 * 16 * 2 * at.heads * at.dim_head * 2
    step = model.engine.KV_CACHE_STEP
    bound = peak8 + 56 * kv + (64 - step) * kv + (2 << 20)
    assert dec.captures == 1 and peak64 <= bound, (peak8, peak64, kv, (peak64 - peak8) / kv)
