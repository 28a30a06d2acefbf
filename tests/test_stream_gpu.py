"""Streaming tokenize / decode (magvit2_pytorch_b200/stream.py) on the device: chunked pushes against one whole-clip call,
bit for bit.  Run on the H100 box:  python -m pytest tests -m gpu"""
import pytest
import torch

from oracle import weights as W
from tests.util import README_LAYERS, build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu

CONFIGS = ["mini", "mini_gateloop", "mini_cond", "mini_sff", "mini_mc", "mini_fsq", "mini_noff"]


def _model(name, dtype):
    assert torch.cuda.is_available(), "gpu-marked test without a GPU"
    g = load_golden(name)
    return g, build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)


def _schedules(tdf, n_lat, ff):
    """Encoder chunk schedules (frame counts) for a clip of n_lat latent frames: whole clip, first frame then tdf frames per
    push, first frame then 2 tdf then tdf, ... (without a first frame: tdf-multiples only)."""
    head = [1] if ff else []
    rest = n_lat - 1 if ff else n_lat
    total = sum(head) + rest * tdf
    scheds = [[total], head + [tdf] * rest]
    if rest >= 3:
        scheds.append(head + [2 * tdf] + [tdf] * (rest - 2))
    return scheds


def _tokenize_stream(model, video, sched, cond=None, ff=True):
    enc = model.tokenize_stream(batch_size=video.shape[0], cond=cond, video_contains_first_frame=ff)
    outs, t = [], 0
    for n in sched:
        outs.append(enc.push(video[:, :, t:t + n]))
        t += n
    return torch.cat(outs, dim=1)


def _decode_stream(model, codes, sizes, cond=None, ff=True):
    dec = model.decode_stream(batch_size=codes.shape[0], cond=cond, video_contains_first_frame=ff)
    outs, t = [], 0
    for n in sizes:
        outs.append(dec.push(codes[:, t:t + n]))
        t += n
    return torch.cat(outs, dim=2)


def _one_shot(model, video, cond, ff):
    codes = model(video, cond=cond, return_codes=True, video_contains_first_frame=ff)
    recon = model.decode_from_code_indices(codes, cond=cond, video_contains_first_frame=ff)
    return codes, recon


def _check_stream_equals_one_shot(model, video, cond, ff, n_lat):
    tdf = model.time_downsample_factor
    codes, recon = _one_shot(model, video, cond, ff)
    assert codes.shape[1] == n_lat
    for sched in _schedules(tdf, n_lat, ff):
        assert torch.equal(_tokenize_stream(model, video, sched, cond, ff), codes), sched
    for sizes in ([n_lat], [1] * n_lat, [1, 2] + [1] * (n_lat - 3)):
        got = _decode_stream(model, codes, sizes, cond, ff)
        assert got.dtype == recon.dtype and torch.equal(got, recon), sizes
    return codes, recon


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", CONFIGS)
def test_stream_equals_one_shot(name, dtype):
    g, model = _model(name, dtype)
    ff = name != "mini_noff"
    tdf = model.time_downsample_factor
    n_lat = 4
    T = (1 + (n_lat - 1) * tdf) if ff else n_lat * tdf
    video = W.synth_video(2, 3, T, model.image_size, seed=11).cuda()
    cond = g["cond"].cuda() if model.has_cond else None
    _check_stream_equals_one_shot(model, video, cond, ff, n_lat)


@pytest.mark.parametrize("name", CONFIGS)
def test_stream_fp32_codes_equal_golden(name):
    """The golden clip streamed one latent frame's worth per push gives the reference's codes."""
    g, model = _model(name, torch.float32)
    ff = name != "mini_noff"
    video = golden_video(g).cuda()
    tdf = model.time_downsample_factor
    n_lat = g["codes"].shape[1]
    sched = ([1] + [tdf] * (n_lat - 1)) if ff else [tdf] * n_lat
    cond = g["cond"].cuda() if model.has_cond else None
    assert torch.equal(_tokenize_stream(model, video, sched, cond, ff).cpu(), g["codes"])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_stream_readme_config(dtype):
    """README config (random weights), two distinct clips at 128^2: every slab / fused-ResidualUnit / conv_out path."""
    torch.manual_seed(0)
    kw = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    model = build_product(kw, 3).cuda().to(dtype)
    video = W.synth_video(2, 3, 13, 128, seed=5).cuda()
    _check_stream_equals_one_shot(model, video, None, True, 4)
    if dtype == torch.bfloat16:
        assert model.engine.fused_ru_calls > 0 and model.engine.slab_calls > 0


def test_stream_uint8_frames():
    g, model = _model("mini", torch.bfloat16)
    video = (W.synth_video(2, 3, 9, 32, seed=3) * 127 + 128).clamp(0, 255).to(torch.uint8).cuda()
    codes = model.tokenize(video)
    assert torch.equal(_tokenize_stream(model, video, [1, 4, 4]), codes)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_long_stream(dtype):
    """16 latent frames, one per push.  In bf16 the whole-clip call runs the general time-attention kernel at L = 16 while
    the pushes up to L = 8 ran the short-sequence one on their rows; on this clip both give the same codes and frames
    (measured: 0 tokens differ, recon max-abs 0), so the test holds both dtypes to bit equality."""
    g, model = _model("mini", dtype)
    n_lat = 16
    video = W.synth_video(2, 3, 1 + (n_lat - 1) * 4, 32, seed=7).cuda()
    codes, recon = _one_shot(model, video, None, True)
    s_codes = _tokenize_stream(model, video, [1] + [4] * (n_lat - 1))
    s_recon = _decode_stream(model, codes, [1] * n_lat)
    assert torch.equal(s_codes, codes) and torch.equal(s_recon, recon)


def test_interleaved_streams_and_one_shot_calls():
    g, model = _model("mini_gateloop", torch.float32)
    va = W.synth_video(2, 3, 9, 32, seed=1).cuda()
    vb = W.synth_video(2, 3, 9, 32, seed=2).cuda()
    ref_a, ref_b = model.tokenize(va), model.tokenize(vb)
    ea, eb = model.tokenize_stream(batch_size=2), model.tokenize_stream(batch_size=2)
    outs_a, outs_b = [], []
    for t0, n in ((0, 1), (1, 4), (5, 4)):
        outs_a.append(ea.push(va[:, :, t0:t0 + n]))
        assert torch.equal(model.tokenize(vb), ref_b)          # a one-shot call between pushes
        outs_b.append(eb.push(vb[:, :, t0:t0 + n]))
    assert torch.equal(torch.cat(outs_a, 1), ref_a) and torch.equal(torch.cat(outs_b, 1), ref_b)


def test_chunk_rule_and_parameter_change_raise():
    g, model = _model("mini", torch.float32)
    enc = model.tokenize_stream(batch_size=2)
    v = W.synth_video(2, 3, 9, 32, seed=1).cuda()
    with pytest.raises(ValueError, match="1 \\+ k"):
        enc.push(v[:, :, :4])
    enc.push(v[:, :, :1])
    with pytest.raises(ValueError, match="k \\* 4"):
        enc.push(v[:, :, 1:3])
    with pytest.raises(ValueError, match="batch"):
        enc.push(v[:1, :, 1:5])
    enc.push(v[:, :, 1:5])
    with torch.no_grad():
        model.conv_in.conv.weight.mul_(1.0)                     # an in-place edit: the packs are rebuilt
    with pytest.raises(RuntimeError, match="parameters changed"):
        enc.push(v[:, :, 5:9])
    dec = model.decode_stream(batch_size=2)
    with pytest.raises(ValueError, match="at least one latent frame"):
        dec.push(torch.zeros((2, 0, 4, 4), dtype=torch.long, device="cuda"))


def test_decode_stream_memory_grows_with_the_kv_cache_only():
    """README config: after 8 latent frames the peak allocation of further one-frame pushes grows by the time attention's
    K/V cache only, not with the clip."""
    torch.manual_seed(0)
    kw = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    model = build_product(kw, 3).cuda().to(torch.bfloat16)
    codes = torch.randint(0, 1024, (1, 64, 16, 16), device="cuda")
    dec = model.decode_stream(batch_size=1)
    for i in range(8):
        dec.push(codes[:, i:i + 1])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for i in range(8, 16):
        dec.push(codes[:, i:i + 1])
    peak8 = torch.cuda.max_memory_allocated()
    for i in range(16, 64):
        dec.push(codes[:, i:i + 1])
    peak64 = torch.cuda.max_memory_allocated()
    # K/V bytes of one latent frame of the single attend_time block: 16 x 16 pixels x 2 x heads * dim_head bf16 (0.25 MiB)
    at = model.decoder_layers[0][0].fn.fn
    kv = 16 * 16 * 2 * at.heads * at.dim_head * 2
    step = model.engine.KV_CACHE_STEP
    # 56 more frames (8 -> 64) in the cache, plus what its growth adds on top: while the cache grows from 64 - step to 64
    # frames the old buffer stays alive until it has been copied into the new one (the capacity is a multiple of `step`, so
    # both peaks see a rounded cache).  Slack: 2 MiB of allocator rounding.
    bound = peak8 + 56 * kv + (64 - step) * kv + (2 << 20)
    assert peak64 <= bound, (peak8, peak64, kv, (peak64 - peak8) / kv)
