"""The video's data gradient (the gradient of a differentiable encode with respect to its video, through conv_in or its
first-frame conv) against float64, on every kernel it runs on: one TrainRunner call at a time, then every such call of a
differentiable encode at the README shape.

The call.  TrainRunner._video_dgrad(g, weight, k, t_crop) is the transposed conv of conv_in: g (B, Ti, H, W, init_dim)
channels-last, the module-layout weight (init_dim, channels, *k) flipped and transposed by transposed_pack, output torch's
(B, channels, Ti - t_crop, H, W) without the t_crop time-padding frames.  bf16 runs it on the slab kernel's channels-first
flavour (the narrow 8- / 16-column N tiles for 7- and 5-wide taps, the ragged 32-column tile for 3x3x3) with a negative
leading time pad, and otherwise channels-last on the CUDA-core, tap-wise or slab conv plus a layout pass: the route table
of tests/test_slab_plan_narrow.py, which each case asserts along with the slab plan's bn and mw.

Part 1, one call at a time.  Outputs start NaN-filled between sentinels (_Guard of tests/test_conv_forward_gpu.py).
  * Real data: each clip against float64 autograd of the forward conv the engine runs (the video behind t_crop zero
    frames, causal zero pad of kt - 1 frames, symmetric H / W pad), alone, so a read of the next clip's frames fails.  The
    bound is the other call tests': half an ulp plus gamma(K, C_OF[kernel]) (|g| (*) |w|), K = init_dim x taps.
  * Exact replay of every slab case on REPLAY_GRID operands (tests/test_bench_calls_gpu.py): up to depth 128 x 343 =
    43904 the products are multiples of 2^-8 of size <= 1/4, so every partial sum is below 2^14 and exact in fp32
    (tests/test_bench_calls_cpu.py); the only allowance left is the output's bf16 rounding.  Where the last tile's CTA ran
    an earlier tile (every case of VIDEO_DGRAD_SLAB), the bound rejects, at the schedule's last tile, one ring stage missing
    (frame tap 0: the transposed conv reads forward in time) and that tile's accumulators not reset (_defect_deltas).
  * Negative controls, each rejected by the bound the kernel passes: time taps not flipped; t_crop off by one (cropped one
    frame late); clip b + 1's leading frames of g read as clip b's frames past its end; the in-plane taps flipped in h only.

Part 2, every video-gradient call of a differentiable encode.  Models built as bench.py builds them (README_KW, synth_data
weights, bf16, eval, use_gan False, no perceptual loss), 4 fp32 clips of 17 x 128^2 (16 frames without a first frame)
that require grad; README with and without a first frame, separate_first_frame_encoding, 12, 1 and 8 channels, and
pad_mode 'reflect'.  TrainRunner.video_dgrad_packed and _conv_bwd_padmode are wrapped: each call is checked against float64
from the module's own weight when it returns.  video.grad must then equal the recorded outputs placed at their frames,
bit for bit after the cast to the video's dtype; the time-padding frames are left out; the separate first frame comes
from conv_in_first_frame, and a first frame taken from the causal conv_in weight is rejected.  The 'reflect' data
gradient is cuDNN's, folded back through F.pad in bf16: each padded element is one of at most 2 x 2 x 2 terms (time, h,
w) added in bf16, so its bound adds 8 bf16 half-ulps of the fold of |g| (*) |w| to the accumulation allowance."""
import math
import time

import pytest
import torch
import torch.nn.functional as F

import synth_data
from bench import README_KW
from tests.test_bench_calls_gpu import _defect_deltas, _grid, _lib_plan, _n_sm
from tests.test_conv_forward_gpu import _Guard, _ran
from tests.test_conv_grad_gpu import C_OF, _gamma
from tests.test_simt_ops_gpu import _check, _rejects
from tests.test_slab_plan_narrow import K177, K333, K555, K777, VIDEO_DGRAD_SLAB, _want

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.train import TrainRunner, transposed_pack

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
STAGE, RESET = "one ring stage missing", "previous tile's accumulators not reset"
NOT_FLIPPED, CROP, BLEED, H_FLIP = ("time taps not flipped", "t_crop off by one", "clip b+1 read past clip b's end",
                                    "in-plane taps flipped in h only")
U_BF = 2.0 ** -9                       # half an ulp of bf16, relative


def _require_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


# ---------------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------------
def _vgrad_full64(g, w, k):
    """float64 gradient wrt x (B, C, Ti, H, W) of conv3d(x behind a causal zero pad of kt - 1 frames, symmetric H / W pad;
    w (init_dim, C, *k) in module layout) for the cotangent g (B, Ti, H, W, init_dim) channels-last."""
    kt, kh, kw = k
    w5 = w.double().reshape(w.shape[0], -1, kt, kh, kw)
    B, Ti, H, W, _ = g.shape
    x = torch.zeros((B, w5.shape[1], Ti, H, W), device="cuda", dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        y = F.conv3d(F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0)), w5)
        gx, = torch.autograd.grad(y, x, g.double().permute(0, 4, 1, 2, 3))
    return gx


def _vgrad64(g, w, k, t_crop):
    """The video's gradient: _vgrad_full64 without the first t_crop frames (the video behind t_crop zero frames)."""
    return _vgrad_full64(g, w, k)[:, :, t_crop:]


def _bound(g, w, k, t_crop, kind):
    """The accumulation allowance gamma(K, c) (|g| (*) |w|) of a real-data call, K = init_dim x taps."""
    return _gamma(w.shape[0] * math.prod(k), C_OF[kind]) * _vgrad64(g.abs(), w.abs(), k, t_crop)


def _padmode_grad64(g, x, w, k, mode):
    """float64 gradient wrt x (B, Ti, H, W, C) channels-last of conv3d(F.pad(x, causal kt - 1, symmetric H / W, mode), w)
    for the cotangent g (B, Ti, H, W, init_dim)."""
    kt, kh, kw = k
    x_ = x.double().permute(0, 4, 1, 2, 3).detach().requires_grad_(True)
    with torch.enable_grad():
        y = F.conv3d(F.pad(x_, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0), mode=mode), w.double())
        gx, = torch.autograd.grad(y, x_, g.double().permute(0, 4, 1, 2, 3))
    return gx.permute(0, 2, 3, 4, 1)


# ---------------------------------------------------------------------------------------------------------------------------
# part 1: one _video_dgrad call at a time
# ---------------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _runner(dtype):
    """A TrainRunner on a small tokenizer's engine (the call reads only the engine), one per dtype."""
    if dtype not in _MODELS:
        m = VideoTokenizer(image_size=32, init_dim=64, codebook_size=1024, layers=("residual", "compress_time"),
                           use_gan=False, perceptual_loss_weight=0.)
        _MODELS[dtype] = m.cuda().to(dtype)
    return TrainRunner(_MODELS[dtype])


def _kcase(name, dtype, shape, kind):
    return pytest.param(name, dtype, shape, kind, id=f"{name}-{'bf16' if dtype == BF else 'fp32'}")


# (B, Ti, t_crop, H, W, init_dim, channels, k), Ti counting the time-padding frames.  Small-frame edges, one tile per CTA:
# T = 1 with and without a time-padding frame, frame sizes that are not tile multiples, B > 1, the first-frame conv
EDGES = {"t1": (1, 1, 0, 16, 16, 64, 3, K777), "t1_tpad": (1, 2, 1, 16, 16, 64, 3, K777),
        "b2_20x27": (2, 4, 1, 20, 27, 64, 3, K777), "r13x9": (1, 2, 0, 13, 9, 64, 3, K777),
        "ff_b2_21x18": (2, 2, 1, 21, 18, 64, 3, K177), "ff_16x40": (1, 1, 0, 16, 40, 64, 3, K177)}
KCASES = ([_kcase(n, BF, s, "slab") for n, (s, _) in VIDEO_DGRAD_SLAB.items()] + [
    _kcase("c8_k777", BF, (4, 20, 3, 128, 128, 64, 8, K777), "simt"),
    _kcase("c16_k777", BF, (4, 20, 3, 128, 128, 64, 16, K777), "simt"),
    _kcase("c8_k555", BF, (2, 20, 3, 64, 64, 64, 8, K555), "simt"),
    _kcase("c8_first_frame", BF, (4, 1, 0, 128, 128, 64, 8, K177), "tap"),
    _kcase("c16_first_frame", BF, (4, 1, 0, 128, 128, 64, 16, K177), "tap"),
    _kcase("c8_k333", BF, (4, 20, 3, 128, 128, 64, 8, K333), "slab"),
    _kcase("readme", F32, VIDEO_DGRAD_SLAB["readme"][0], "simt")] +
    [_kcase(n, dt, s, "slab" if dt == BF else "simt") for n, s in EDGES.items() for dt in (BF, F32)])


def _controls(out, g, w, k, t_crop, dtype, acc):
    """The negative controls that apply to the call, each rejected by the bound clip 0 passes -> their names."""
    kt = k[0]
    w5 = w.reshape(w.shape[0], -1, *k)
    g0 = g[:1].double()
    full = _vgrad_full64(g0, w5, k)
    wrong = {H_FLIP: _vgrad64(g0, w5.flip(3), k, t_crop),
             CROP: torch.cat((full[:, :, t_crop + 1:], torch.zeros_like(full[:, :, :1])), 2)}
    if kt > 1:
        wrong[NOT_FLIPPED] = _vgrad64(g0, w5.flip(2), k, t_crop)
        if g.shape[0] > 1:
            Ti = g.shape[1]
            wrong[BLEED] = _vgrad_full64(g[:2].double().reshape(1, 2 * Ti, *g.shape[2:]), w5, k)[:, :, t_crop:Ti]
    for name, ref in wrong.items():
        _rejects(out[:1], ref, dtype, acc, f"control: {name}")
    return sorted(wrong)


@pytest.mark.parametrize("name,dtype,shape,kind", KCASES)
def test_video_dgrad_vs_float64(monkeypatch, name, dtype, shape, kind):
    _require_cuda()
    B, Ti, t_crop, H, W, D, Cv, k = shape
    kt, kh, kw = k
    To = Ti - t_crop
    runner = _runner(dtype)
    eng = runner.eng
    guard = _Guard(eng)
    monkeypatch.setattr(eng, "_new", guard.new)
    monkeypatch.setattr(eng, "conv_log", [])
    gen = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    wshape = (D, Cv, kh, kw) if k == K177 else (D, Cv, *k)            # Conv2d / Conv3d module layout
    w = (torch.randn(wshape, generator=gen, device="cuda") * 0.05).to(dtype)
    g = torch.randn((B, Ti, H, W, D), generator=gen, device="cuda").to(dtype)

    def call(g_, w_):
        n0 = len(guard.allocs)
        ran, out = _ran(eng, lambda: runner._video_dgrad(g_, w_, k, t_crop))
        guard.check_borders(name)
        del guard.allocs[n0:]
        assert out.shape == (B, Cv, To, H, W) and out.dtype == dtype
        return ran, out

    ran, out = call(g, w)
    assert ran == kind == _want(dtype, Cv, k)[0], f"{name}: ran {ran}, expected {kind}"
    pk = transposed_pack(w, k, dtype)
    cf = dtype == BF and eng.conv_cf_supported(g, pk, (-t_crop, kh // 2, kw // 2), (To, H, W))
    assert cf == _want(dtype, Cv, k)[1]
    info = f"{name}: {ran}{' channels-first' if cf else ' + layout pass'}"
    plan = None
    if cf:
        ta = eng._tc_args(g, pk, pad=(-t_crop, kh // 2, kw // 2), out_spatial=(To, H, W), out_cf=True)
        plan = _lib_plan(eng.lib, ta, _n_sm())
        if name in VIDEO_DGRAD_SLAB:
            bn, mw, _ = VIDEO_DGRAD_SLAB[name][1]
            assert (plan["bn"], plan["mw"]) == (bn, mw), plan
            assert plan["total"] > plan["grid"], plan
        info += f", bn {plan['bn']}, mw {plan['mw']}, {plan['total']} tiles = {-(-plan['total'] // plan['grid'])} per CTA"
    # ---- real data, one clip at a time ----
    acc0 = None
    for i in range(B):
        acc = _bound(g[i:i + 1], w, k, t_crop, ran)
        _check(out[i:i + 1], _vgrad64(g[i:i + 1], w, k, t_crop), dtype, acc, f"{name}, clip {i}")
        if i == 0:
            acc0 = acc
    controls = _controls(out, g, w, k, t_crop, dtype, acc0)
    info += f"; controls rejected: {controls}"
    # ---- exact replay, the pipeline defects at the schedule's last tile ----
    if cf:
        gr, wr = _grid((B, Ti, H, W, D), "x", gen), _grid(wshape, "w", gen)
        ran2, outr = call(gr.to(BF), wr.to(BF))
        assert ran2 == ran
        refs = [_vgrad64(gr[i:i + 1], wr, k, t_crop) for i in range(B)]
        for i in range(B):
            _check(outr[i:i + 1], refs[i], BF, 0, f"{name}: replay, clip {i}")
        rejected = []
        if plan["total"] > plan["grid"]:
            wt = wr.reshape(D, Cv, *k).flip(2, 3, 4).transpose(0, 1)        # the transposed conv's (Co, Ci) weight
            for defect, (b, delta) in _defect_deltas(eng.lib, ta, _n_sm(), lambda i: gr[i:i + 1], wt,
                                                     (-t_crop, kh // 2, kw // 2), (To, H, W), None, plan).items():
                _rejects(outr[b:b + 1], refs[b] + delta.permute(0, 4, 1, 2, 3), BF, 0, f"{name}: {defect}")
                rejected.append(defect)
            assert sorted(rejected) == sorted([STAGE, RESET])
        info += f"; replayed exactly, defects rejected: {rejected}"
    print(info)


# ---------------------------------------------------------------------------------------------------------------------------
# part 2: every video-gradient call of a differentiable encode at the README shape
# ---------------------------------------------------------------------------------------------------------------------------
ENCODE_CONFIGS = {"readme": ({}, True), "readme_no_first_frame": ({}, False),
                  "sff": (dict(separate_first_frame_encoding=True), True), "c12": (dict(channels=12), True),
                  "c1": (dict(channels=1), True), "c8": (dict(channels=8), True), "reflect": (dict(pad_mode="reflect"), True)}


def _encode_model(extra):
    torch.manual_seed(0)
    m = VideoTokenizer(**README_KW, use_gan=False, perceptual_loss_weight=0., **extra)
    synth_data.fill_state_dict_(m, 0)
    return m.cuda().bfloat16().eval()


@pytest.mark.parametrize("config", sorted(ENCODE_CONFIGS))
def test_encode_video_gradient_calls(monkeypatch, config):
    _require_cuda()
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    extra, ff = ENCODE_CONFIGS[config]
    m = _encode_model(extra)
    eng = m.engine
    Cv, t_pad = m.channels, m.time_padding if ff else 0
    sff = m.separate_first_frame_encoding and ff
    kin = tuple(m.conv_in.conv.weight.shape[2:])
    T = 17 if ff else 16
    calls, padmode = [], []
    orig, orig_p = TrainRunner.video_dgrad_packed, TrainRunner._conv_bwd_padmode
    monkeypatch.setattr(eng, "conv_log", [])

    def video_dgrad_packed(runner, g, pk, t_crop):
        ran, out = _ran(eng, lambda: orig(runner, g, pk, t_crop))
        torch.cuda.synchronize()
        k = tuple(pk.k)
        first = k[0] == 1 and sff
        w = (m.conv_in_first_frame if first else m.conv_in.conv).weight
        assert ran == _want(BF, Cv, k)[0], (config, k, ran)
        what = f"{config}: video dgrad k{k} t_crop {t_crop} on {ran}"
        accs = []
        for i in range(g.shape[0]):
            accs.append(_bound(g[i:i + 1], w, k, t_crop, ran))
            _check(out[i:i + 1], _vgrad64(g[i:i + 1], w, k, t_crop), BF, accs[-1], f"{what}, clip {i}")
        calls.append(dict(k=k, t_crop=t_crop, out=out.clone(), g=g.clone(), kind=ran, first=first, acc0=accs[0]))
        return out

    def conv_bwd_padmode(runner, g, x, weight, bias, k, pad_mode, need_gx=True):
        out = orig_p(runner, g, x, weight, bias, k, pad_mode, need_gx)
        if runner.m is m and weight is m.conv_in.conv.weight and need_gx:
            torch.cuda.synchronize()
            assert pad_mode != "constant" and out.shape == x.shape, (pad_mode, out.shape)
            ref = _padmode_grad64(g, x, weight, k, pad_mode)
            S = _padmode_grad64(g.abs(), x, weight.abs(), k, pad_mode)
            acc = (_gamma(weight.shape[0] * math.prod(k), C_OF["cudnn"]) + 8 * U_BF * 1.01) * S
            _check(out, ref, BF, acc, f"{config}: conv_in data gradient through F.pad({pad_mode})")
            padmode.append(dict(out=out.clone(), t_pad=x.shape[1] - T))
        return out

    monkeypatch.setattr(TrainRunner, "video_dgrad_packed", video_dgrad_packed)
    monkeypatch.setattr(TrainRunner, "_conv_bwd_padmode", conv_bwd_padmode)
    video = synth_data.synth_video(4, Cv, T, 128, seed=1000).cuda().requires_grad_(True)
    out = m.encode(video, video_contains_first_frame=ff)
    r = torch.randn(out.shape, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    (out.float() * r).sum().backward()
    torch.cuda.synchronize()
    gv = video.grad
    assert gv is not None and gv.dtype == video.dtype and gv.shape == video.shape
    # ---- assembly: video.grad is the recorded outputs at their frames, the time padding left out ----
    if m.conv_in.pad_mode != "constant":
        assert not calls and len(padmode) == 1
        assert padmode[0]["t_pad"] == t_pad == 3
        assert torch.equal(gv, padmode[0]["out"][:, t_pad:].permute(0, 4, 1, 2, 3).to(video.dtype))
        placed = "the F.pad fold's frames 3.."
    elif sff:
        assert not padmode and [(c["k"], c["t_crop"], c["first"]) for c in calls] == [((1,) + kin[1:], 0, True), (kin, 0, False)]
        c0, c1 = calls
        assert c0["g"].shape[1] == 1 and c1["g"].shape[1] == T - 1
        assert torch.equal(gv[:, :, :1], c0["out"].to(video.dtype)) and torch.equal(gv[:, :, 1:], c1["out"].to(video.dtype))
        # control: the first frame's gradient taken from the causal conv_in weight over the encoder's 17 frames
        g_all = torch.cat((c0["g"], c1["g"]), 1)
        wrong = _vgrad64(g_all[:1], m.conv_in.conv.weight, kin, 0)[:, :, :1]
        _rejects(gv[:1, :, :1], wrong, BF, c0["acc0"], f"{config}: control: first frame from the causal conv_in weight")
        placed = "frame 0 from conv_in_first_frame, frames 1.. from conv_in"
    else:
        assert not padmode and len(calls) == 1
        c = calls[0]
        assert (c["k"], c["t_crop"]) == (kin, t_pad) and c["g"].shape[1] == T + t_pad
        assert torch.equal(gv, c["out"].to(video.dtype))
        placed = f"one call, t_crop {t_pad}"
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"{config}: {[(c['k'], c['kind']) for c in calls] or 'cuDNN + F.pad fold'}; video.grad bit for bit = {placed}; "
          f"wall {time.time() - t0:.1f} s, peak device memory {peak:.1f} GiB")
