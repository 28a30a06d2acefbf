"""The training backward's conv data gradients ("dgrad": the gradient wrt a conv's input) on the engine's conv kernels, and the
layout choices around the weight / bias gradients of aten.convolution_backward, against plain float64 torch references.

  A. TapeRunner._dgrad (every stride-1 causal conv: the ResidualUnit 3x3x3 and 1x1x1 convs, conv_out, the discriminator's
     3x3 and 1x1 convs) and DiscrRunner._dgrad_s2 (the discriminator's stride-2 convs as a 1x1 conv with the depth-to-space
     store) on the slab kernel (tc_slab.cu), the tap-wise kernel (tc_conv.cu) and the CUDA-core conv (simt_ops.cu), at the
     edges only the backward reaches: gx[t] = sum_e W'[e] g[t + e] reads frames past the end of the clip, which every kernel
     must read as zeros without touching the next clip.  Each case asserts from the engine's counters which kernel ran.
  B. TapeRunner._conv_bwd / TrainRunner._conv_bwd_padmode in fp32: the front time pad of a channels-last tensor, the
     channels-first conv_in input with its time_padding, the separate first-frame conv and the reflect / replicate /
     circular pad modes (with their fallback to zero padding) against float64 autograd of the same conv.
  C. Every dgrad call of a bf16 and an fp32 generator step of the README config and of a bf16 discriminator step, recorded
     and checked one by one, with the number of calls the model's stages imply.

References.  The reference of a data gradient is torch.autograd.grad, in float64, of the forward the engine runs
(oracle.restated.causal_conv3d, or F.conv2d of the pixel-unshuffled / strided input), so a wrong flip or pad on the host
side fails as well as a kernel defect.  Synthetic operands are bf16-representable, so kernel and reference see the same
values.

Error bounds (per element).  Half an ulp of the output dtype at the reference value (the single rounding of the fp32
accumulator) plus an fp32 accumulation allowance gamma * (|W| (*) |g|), where (|W| (*) |g|) is the same gradient of absolute
values in float64, K the summation depth (Co * kt * kh * kw for a data gradient, B * To * Ho * Wo for a weight / bias
gradient) and gamma = c K u / (1 - c K u), u = 2^-24.  A sum of K products whose every operation rounds to nearest, in any
order, is within gamma(c = 1) of the exact sum (Higham, Accuracy and Stability, 3.1 / 3.5); the fp32 products of bf16
operands are exact.
  * CUDA-core conv: per-thread fp32 fma chains, round to nearest: c = 1.
  * wgmma kernels: the tensor core adds its exact bf16 products in fp32 without a guarantee of round-to-nearest (it may
    truncate the aligned addends), so each addition may lose up to 2u: c = 2.
  * cuDNN (weight / bias gradients, strided data gradients; TF32 off): its algorithm, and so its order, is its own choice;
    c = 2 as for an adder that truncates.
Each family also shows that its bound rejects a slightly wrong reference (time taps not flipped, the gradient one frame
late, clip 1 bled into clip 0, a spatial tap dropped, swapped depth-to-space phases, the time pad at the back, the
first-frame conv's gradient taken from frame 1), so a kernel or host defect of that kind would fail."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R
from tests.test_simt_ops_gpu import U, _check, _rejects
from tests.util import README_LAYERS, build_product, golden_video, load_golden

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.gan import DiscrRunner, stride2_1x1_dgrad_weight, unshuffle_dgrad_weight
from magvit2_pytorch_b200.train import TapeRunner, TrainRunner

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "f32": torch.float32}
C_OF = {"simt": 1, "tap": 2, "slab": 2, "cudnn": 2}       # c of the accumulation allowance, per summation order (see above)


@pytest.fixture(autouse=True)
def _no_tf32():
    """cuDNN in true fp32 (TF32 would round far above fp32 round-off); restored even when a test fails."""
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


# ------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(dtype):
    """A small tokenizer whose engine runs the conv calls (as test_tc_conv_gpu._engine), one per dtype."""
    if dtype not in _MODELS:
        _MODELS[dtype] = VideoTokenizer(image_size=32, init_dim=16, codebook_size=1024, layers=("residual",)).cuda().to(dtype)
    return _MODELS[dtype]


def _engine(dtype, variant):
    """variant "auto": the slab kernel where it takes the shape, else the tap-wise one; "tap": the tap-wise kernel;
    "simt": the CUDA-core conv (use_tc off).  An fp32 engine always runs the CUDA-core conv."""
    eng = _model(dtype).engine
    eng.use_tc = variant != "simt"
    eng.tc_variant = "tap" if variant == "tap" else "auto"
    return eng


def _gen(name):
    return torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))


def _bfrand(shape, g, scale=1.0):
    """bf16-representable normal values, as float64."""
    return (torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) * scale).to(torch.bfloat16).double()


def _launch(eng, fn):
    """(kernel that ran, result) of one conv call, from the engine's counters."""
    def counts():
        return eng.slab_calls, eng.tc_calls, eng.simt_conv_calls
    c0 = counts()
    out = fn()
    d = tuple(a - b for a, b in zip(counts(), c0))
    return {(1, 1, 0): "slab", (0, 1, 0): "tap", (0, 0, 1): "simt"}.get(d, f"counters moved by {d}"), out


def _gamma(K, c):
    return c * K * U / (1 - c * K * U)


def _dgrad64(g, w, k, out_spatial):
    """float64 gradient wrt its input of the conv the engine runs forward, y = conv(x; w) with leading pad
    (kt - 1, kh // 2, kw // 2) (R.causal_conv3d).  g (B,To,Ho,Wo,Co) channels-last -> (B,T,H,W,Ci) channels-last."""
    kt, kh, kw = k
    w5 = w.double().reshape(w.shape[0], -1, kt, kh, kw)
    x = torch.zeros((g.shape[0], w5.shape[1], *out_spatial), device="cuda", dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        gx, = torch.autograd.grad(R.causal_conv3d(x, w5, None), x, g.double().permute(0, 4, 1, 2, 3))
    return gx.permute(0, 2, 3, 4, 1)


def _s2_grad64(g, w, stride2_1x1, hw):
    """float64 gradient wrt h of F.conv2d(F.pixel_unshuffle(h, 2), w) (w: (Co, 4 Ci, 1, 1)) or, stride2_1x1, of the 1x1
    stride-2 F.conv2d(h, w) (w: (Co, Ci, 1, 1)).  g (B,1,Ho,Wo,Co) -> (B,1,H,W,Ci) channels-last."""
    ci = w.shape[1] if stride2_1x1 else w.shape[1] // 4
    h = torch.zeros((g.shape[0], ci, *hw), device="cuda", dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        y = F.conv2d(h, w.double(), stride=2) if stride2_1x1 else F.conv2d(F.pixel_unshuffle(h, 2), w.double())
        gh, = torch.autograd.grad(y, h, g.double()[:, 0].permute(0, 3, 1, 2))
    return gh.permute(0, 2, 3, 1)[:, None]


# ------------------------------------------------------------------------------------------------------------------
# A. TapeRunner._dgrad at the kernels' edges
# ------------------------------------------------------------------------------------------------------------------
K333, K111, K133 = (3, 3, 3), (1, 1, 1), (1, 3, 3)
DG_CASES = [
    # name, dtype, variant, forward Ci, forward Co, k, (B, T, H, W), kernel that must run.  The dgrad conv reads Co channels
    # and writes Ci: 16 channels take the tap-wise kernel's 32-byte rows, 32 the slab's 64-byte rows (kw = 1 only), 48 is
    # not a multiple of 32.  B = 2 cases scale clip 1's gradient by 8.
    ("slab_c64_k333_T5", "bf16", "auto", 64, 64, K333, (2, 5, 16, 16), "slab"),
    ("slab_c64_k333_T1", "bf16", "auto", 64, 64, K333, (2, 1, 16, 16), "slab"),
    ("slab_c64_k333_T2_24x20", "bf16", "auto", 64, 64, K333, (2, 2, 24, 20), "slab"),
    ("slab_c64_k333_T3_12x40", "bf16", "auto", 64, 64, K333, (1, 3, 12, 40), "slab"),
    ("slab_c64_k333_T2_w128", "bf16", "auto", 64, 64, K333, (2, 2, 8, 128), "slab"),
    ("slab_c64_k333_320tiles", "bf16", "auto", 64, 64, K333, (2, 5, 128, 128), "slab"),
    ("slab_c128_k333_T3_20x24", "bf16", "auto", 128, 128, K333, (2, 3, 20, 24), "slab"),
    ("slab_c256_k333_T2", "bf16", "auto", 256, 256, K333, (2, 2, 16, 16), "slab"),
    ("slab_c512_k333_T3", "bf16", "auto", 512, 512, K333, (2, 3, 8, 8), "slab"),
    ("slab_c512_k333_T20", "bf16", "auto", 512, 512, K333, (1, 20, 16, 16), "slab"),
    ("slab_c32_k111_T3", "bf16", "auto", 32, 32, K111, (2, 3, 16, 16), "slab"),
    ("slab_c64_k111_T1", "bf16", "auto", 64, 64, K111, (2, 1, 24, 20), "slab"),
    ("slab_c512_k111_T5", "bf16", "auto", 512, 512, K111, (2, 5, 8, 8), "slab"),
    ("slab_c64_k133_T3_24x20", "bf16", "auto", 64, 64, K133, (2, 3, 24, 20), "slab"),
    ("slab_c512_k133_T1", "bf16", "auto", 512, 512, K133, (2, 1, 8, 8), "slab"),
    ("slab_c256_k133_T1_16x16", "bf16", "auto", 256, 256, K133, (2, 1, 16, 16), "slab"),
    ("discr_image_co64_slab", "bf16", "auto", 3, 64, K133, (2, 1, 32, 32), "slab"),
    ("discr_image_co256_slab", "bf16", "auto", 3, 256, K133, (2, 1, 32, 32), "slab"),
    ("discr_image_co16_tap", "bf16", "auto", 3, 16, K133, (2, 1, 32, 32), "tap"),
    ("tap_c16_k333_T3", "bf16", "auto", 16, 16, K333, (2, 3, 24, 20), "tap"),
    ("tap_c32_k333_T2", "bf16", "auto", 32, 32, K333, (2, 2, 12, 40), "tap"),
    ("tap_c48_k333_T5", "bf16", "auto", 48, 48, K333, (2, 5, 16, 16), "tap"),
    ("tap_c48_k111_T1", "bf16", "auto", 48, 48, K111, (2, 1, 12, 12), "tap"),
    ("tap_c64_k333_T5_24x20", "bf16", "tap", 64, 64, K333, (2, 5, 24, 20), "tap"),
    ("tap_c64_k333_T1", "bf16", "tap", 64, 64, K333, (2, 1, 16, 16), "tap"),
    ("tap_c128_k333_T2_w128", "bf16", "tap", 128, 128, K333, (2, 2, 4, 128), "tap"),
    ("tap_c256_k333_T20", "bf16", "tap", 256, 256, K333, (1, 20, 8, 8), "tap"),
    ("tap_c512_k133_T1", "bf16", "tap", 512, 512, K133, (2, 1, 8, 8), "tap"),
    ("tap_c64_k111_T3", "bf16", "tap", 64, 64, K111, (2, 3, 12, 40), "tap"),
    ("conv_out_bf16", "bf16", "auto", 64, 3, K333, (2, 5, 16, 16), "simt"),
    ("simt_bf16_c64_k333_T2_12x40", "bf16", "simt", 64, 64, K333, (2, 2, 12, 40), "simt"),
    ("simt_bf16_c48_k333_T1", "bf16", "simt", 48, 48, K333, (2, 1, 8, 8), "simt"),
    ("simt_bf16_c16_k133_T3", "bf16", "simt", 16, 16, K133, (2, 3, 24, 20), "simt"),
    ("f32_c64_k333_T5", "f32", "simt", 64, 64, K333, (2, 5, 16, 16), "simt"),
    ("f32_c64_k333_T1", "f32", "simt", 64, 64, K333, (2, 1, 16, 16), "simt"),
    ("f32_c16_k333_T2_24x20", "f32", "simt", 16, 16, K333, (2, 2, 24, 20), "simt"),
    ("f32_c256_k333_T3_12x40", "f32", "simt", 256, 256, K333, (1, 3, 12, 40), "simt"),
    ("f32_c512_k133_T2", "f32", "simt", 512, 512, K133, (2, 2, 8, 8), "simt"),
    ("f32_c128_k111_T3", "f32", "simt", 128, 128, K111, (2, 3, 16, 16), "simt"),
    ("f32_conv_out_T20", "f32", "simt", 64, 3, K333, (1, 20, 16, 16), "simt"),
    ("f32_discr_image_co16", "f32", "simt", 3, 16, K133, (2, 1, 32, 32), "simt"),
]


@pytest.mark.parametrize("name,dt,variant,ci,co,k,shape,kern", DG_CASES, ids=[c[0] for c in DG_CASES])
def test_dgrad_vs_float64(name, dt, variant, ci, co, k, shape, kern):
    dtype = DT[dt]
    eng = _engine(dtype, variant)
    gen = _gen(name)
    B, T, H, W = shape
    kt, kh, kw = k
    w = _bfrand((co, ci, *k), gen, (ci * kt * kh * kw) ** -0.5)          # the forward conv's weight
    g = _bfrand((B, T, H, W, co), gen)
    g[1:] *= 8                                                          # a bleed of clip 1 into clip 0 exceeds the bound
    runner = TapeRunner(eng)
    kind, gx = _launch(eng, lambda: runner._dgrad(g.to(dtype), w.to(dtype), k, (T, H, W)))
    assert kind == kern, f"{name}: expected the {kern} kernel, ran {kind}"
    assert runner.own_dgrad_calls == 1
    assert gx.shape == (B, T, H, W, ci) and gx.dtype == dtype
    ref = _dgrad64(g, w, k, (T, H, W))
    acc = _gamma(co * kt * kh * kw, C_OF[kind]) * _dgrad64(g.abs(), w.abs(), k, (T, H, W))
    _check(gx, ref, dtype, acc, name)
    # the bound rejects slightly wrong references
    wrong = torch.zeros_like(ref)
    wrong[:, 1:] = ref[:, :-1]
    _rejects(gx, wrong, dtype, acc, f"{name}: gradient one frame late")
    if kt > 1:
        _rejects(gx, _dgrad64(g, w.flip(2), k, (T, H, W)), dtype, acc, f"{name}: time taps not flipped")
        if B > 1:          # the clips as one sequence: clip 1's first frames reach clip 0's last kt - 1 frames
            bled = _dgrad64(g.reshape(1, B * T, H, W, co), w, k, (B * T, H, W)).reshape(ref.shape)
            _rejects(gx, bled, dtype, acc, f"{name}: clip 1 bled into clip 0")
    if kh * kw > 1:
        w_drop = w.clone()
        w_drop[:, :, kt - 1, 0, kw - 1] = 0
        _rejects(gx, _dgrad64(g, w_drop, k, (T, H, W)), dtype, acc, f"{name}: one spatial tap dropped")


S2_CASES = [
    # name, dtype, variant, weight builder, forward Ci, forward Co, (B, Ho, Wo), kernel.  The discriminator's channel counts
    # (tests/golden/mini_gan.pt: 3 -> 256 -> 512 -> 512 at 32 -> 16 -> 8 -> 4) plus 16 channels for the tap-wise kernel.
    ("unshuffle_c256_slab", "bf16", "auto", "unshuffle", 256, 256, (2, 8, 8), "slab"),
    ("unshuffle_c512_slab", "bf16", "auto", "unshuffle", 512, 512, (2, 4, 4), "slab"),
    ("unshuffle_c512_tap", "bf16", "tap", "unshuffle", 512, 512, (2, 2, 2), "tap"),
    ("unshuffle_c16_tap", "bf16", "auto", "unshuffle", 16, 16, (2, 16, 16), "tap"),
    ("unshuffle_c256_simt_bf16", "bf16", "simt", "unshuffle", 256, 256, (2, 8, 8), "simt"),
    ("unshuffle_c256_f32", "f32", "simt", "unshuffle", 256, 256, (2, 8, 8), "simt"),
    ("res_s2_c3_bf16", "bf16", "auto", "stride2_1x1", 3, 256, (2, 16, 16), "simt"),
    ("res_s2_c3_f32", "f32", "simt", "stride2_1x1", 3, 256, (2, 16, 16), "simt"),
    ("res_s2_c256_slab", "bf16", "auto", "stride2_1x1", 256, 512, (2, 8, 8), "slab"),
    ("res_s2_c512_tap", "bf16", "tap", "stride2_1x1", 512, 512, (2, 4, 4), "tap"),
    ("res_s2_c512_f32", "f32", "simt", "stride2_1x1", 512, 512, (2, 4, 4), "simt"),
]


def _s2_runner(eng):
    """A DiscrRunner without a discriminator: _dgrad_s2 reads only the engine."""
    r = DiscrRunner.__new__(DiscrRunner)
    TapeRunner.__init__(r, eng)
    return r


@pytest.mark.parametrize("name,dt,variant,builder,ci,co,shape,kern", S2_CASES, ids=[c[0] for c in S2_CASES])
def test_dgrad_stride2_vs_float64(name, dt, variant, builder, ci, co, shape, kern):
    dtype = DT[dt]
    eng = _engine(dtype, variant)
    gen = _gen(name)
    B, Ho, Wo = shape
    one = builder == "stride2_1x1"
    w = _bfrand((co, ci if one else 4 * ci, 1, 1), gen, (ci if one else 4 * ci) ** -0.5)
    wd = (stride2_1x1_dgrad_weight if one else unshuffle_dgrad_weight)(w.to(dtype))
    g = _bfrand((B, 1, Ho, Wo, co), gen)
    g[1:] *= 8
    runner = _s2_runner(eng)
    kind, gx = _launch(eng, lambda: runner._dgrad_s2(g.to(dtype), wd, (B, 1, 2 * Ho, 2 * Wo, ci)))
    assert kind == kern, f"{name}: expected the {kern} kernel, ran {kind}"
    assert runner.own_dgrad_calls == 1 and gx.dtype == dtype
    ref = _s2_grad64(g, w, one, (2 * Ho, 2 * Wo))
    acc = _gamma(co, C_OF[kind]) * _s2_grad64(g.abs(), w.abs(), one, (2 * Ho, 2 * Wo))
    _check(gx, ref, dtype, acc, name)
    if one:        # the only non-zero phase (p1, p2) = (0, 0) stored at (1, 1)
        wrong = torch.zeros_like(ref)
        wrong[:, :, 1::2, 1::2] = ref[:, :, 0::2, 0::2]
        _rejects(gx, wrong, dtype, acc, f"{name}: phase (0, 0) stored at (1, 1)")
    else:
        wrong = ref.reshape(B, 1, Ho, 2, Wo, 2, ci).transpose(3, 5).reshape(ref.shape)
        _rejects(gx, wrong, dtype, acc, f"{name}: p1 and p2 swapped")


# ------------------------------------------------------------------------------------------------------------------
# B. the layouts handed to aten.convolution_backward, fp32
# ------------------------------------------------------------------------------------------------------------------
BWD_CASES = [
    # name, kind, k, stride, pad (None: causal default), Ci, Co, (B, T, H, W), pad mode / time_padding
    ("cl_k333_T5", "cl", K333, (1, 1, 1), None, 16, 24, (2, 5, 10, 12), None),
    ("cl_k333_T2", "cl", K333, (1, 1, 1), None, 16, 24, (2, 2, 10, 12), None),
    ("cl_k333_T1", "cl", K333, (1, 1, 1), None, 16, 24, (2, 1, 10, 12), None),
    ("cl_time_down_T5", "cl", (3, 1, 1), (2, 1, 1), (2, 0, 0), 24, 24, (2, 5, 6, 10), None),
    ("cl_time_down_T1", "cl", (3, 1, 1), (2, 1, 1), (2, 0, 0), 24, 24, (2, 1, 6, 10), None),
    ("cl_space_down", "cl", K133, (1, 2, 2), (0, 1, 1), 16, 32, (2, 3, 12, 10), None),
    ("conv_in_cf_T5", "cf", (7, 7, 7), (1, 1, 1), None, 3, 16, (1, 5, 16, 16), 3),
    ("conv_in_cf_T1", "cf", (7, 7, 7), (1, 1, 1), None, 3, 16, (2, 1, 16, 16), 3),
    ("first_frame", "ff", (1, 7, 7), (1, 1, 1), (0, 3, 3), 3, 16, (2, 5, 16, 16), None),
    ("reflect_T5", "pad", K333, (1, 1, 1), None, 16, 24, (2, 5, 10, 12), "reflect"),
    ("replicate_T3", "pad", K333, (1, 1, 1), None, 16, 24, (2, 3, 10, 12), "replicate"),
    ("circular_T5", "pad", K333, (1, 1, 1), None, 16, 24, (2, 5, 10, 12), "circular"),
    ("reflect_T2_fallback", "pad", K333, (1, 1, 1), None, 16, 24, (2, 2, 10, 12), "reflect"),
    ("circular_T1_fallback", "pad", K333, (1, 1, 1), None, 16, 24, (2, 1, 10, 12), "circular"),
    ("replicate_T1_fallback", "pad", K333, (1, 1, 1), None, 16, 24, (2, 1, 10, 12), "replicate"),
    ("reflect_k777_T8_conv_in", "pad_in", (7, 7, 7), (1, 1, 1), None, 3, 16, (1, 8, 12, 12), "reflect"),
    ("circular_k777_T3_conv_in_fallback", "pad_in", (7, 7, 7), (1, 1, 1), None, 3, 16, (1, 3, 12, 12), "circular"),
]


def _conv64_grads(x, w, b, g, k, stride, pad, mode="constant", back=False):
    """float64 autograd (gx, gw, gb) of y = conv3d(pad(x), w, b, stride): x (B,C,T,H,W), pad (pt, ph, pw) in front of time
    (at the back if `back`) and on both sides of H / W, with F.pad's `mode`.  g (B,To,Ho,Wo,Co) channels-last."""
    pt, ph, pw = pad
    x_, w_, b_ = (t.detach().double().requires_grad_(True) for t in (x, w, b))
    with torch.enable_grad():
        xp = F.pad(x_, (pw, pw, ph, ph) + ((0, pt) if back else (pt, 0)), mode=mode)
        y = F.conv3d(xp, w_.reshape(w.shape[0], -1, *k), b_, stride=stride)
        assert y.shape == g.permute(0, 4, 1, 2, 3).shape, (y.shape, g.shape)
        return torch.autograd.grad(y, (x_, w_, b_), g.double().permute(0, 4, 1, 2, 3))


@pytest.mark.parametrize("name,kind,k,stride,pad,ci,co,shape,extra", BWD_CASES, ids=[c[0] for c in BWD_CASES])
def test_conv_bwd_layouts_vs_float64(name, kind, k, stride, pad, ci, co, shape, extra):
    runner = TrainRunner(_model(torch.float32))
    gen = _gen(name)
    B, T, H, W = shape
    kt, kh, kw = k
    w64 = _bfrand((co, ci, *k) if kind != "ff" else (co, ci, kh, kw), gen, (ci * kt * kh * kw) ** -0.5)
    b64 = _bfrand(co, gen, 0.1)
    wp, bp = torch.nn.Parameter(w64.float()), torch.nn.Parameter(b64.float())
    x64 = video64 = _bfrand((B, ci, T, H, W), gen)                      # channels-first
    x_cl = x64.permute(0, 2, 3, 4, 1).float().contiguous()
    mode, need_gx, gx_by = "constant", True, "cudnn"
    if kind == "cl":
        pad_ = pad if pad is not None else (kt - 1, kh // 2, kw // 2)
        To, Ho, Wo = ((T + pad_[0] - kt) // stride[0] + 1, (H + 2 * pad_[1] - kh) // stride[1] + 1,
                      (W + 2 * pad_[2] - kw) // stride[2] + 1)
        gx_by = "simt" if pad is None else "cudnn"                     # stride-1 causal: the engine's own dgrad
        g64 = _bfrand((B, To, Ho, Wo, co), gen)
        gx = runner._conv_bwd(g64.float().contiguous(), x_cl, wp, bp, k, stride, pad)
    elif kind == "cf":         # conv_in: the channels-first video with time_padding + kt - 1 zero frames in front
        pad_ = (extra + kt - 1, kh // 2, kw // 2)
        need_gx = False
        g64 = _bfrand((B, T + extra, H, W, co), gen)
        gx = runner._conv_bwd(g64.float().contiguous(), x64.float(), wp, bp, k, pad=pad_, need_gx=False, x_is_cf=True)
    elif kind == "ff":         # separate_first_frame_encoding: the first-frame conv on frame 0 of the video
        pad_ = pad
        need_gx = False
        g64 = _bfrand((B, 1, H, W, co), gen)
        gx = runner._conv_bwd(g64.float().contiguous(), x64.float()[:, :, 0:1], wp, bp, k, pad=pad, need_gx=False, x_is_cf=True)
        x64 = x64[:, :, 0:1]
    else:                      # pad modes: the conv_out form (data gradient) and the conv_in form (weights only)
        pad_ = (kt - 1, kh // 2, kw // 2)
        mode = extra if kt - 1 < T else "constant"                  # the forward's fallback (M:925)
        need_gx = kind == "pad"
        gx_by = "cudnn" if mode != "constant" else "simt"
        g64 = _bfrand((B, T, H, W, co), gen)
        gx = runner._conv_bwd_padmode(g64.float().contiguous(), x_cl, wp, bp, k, extra, need_gx=need_gx)
    args = (k, stride, pad_, mode)
    rgx, rgw, rgb = _conv64_grads(x64, w64, b64, g64, *args)
    ax, aw, ab = _conv64_grads(x64.abs(), w64.abs(), b64.abs(), g64.abs(), *args)
    n_out = g64[..., 0].numel()
    acc_w, acc_b = _gamma(n_out, C_OF["cudnn"]) * aw, _gamma(n_out, C_OF["cudnn"]) * ab
    gw, gb = runner.grads[wp], runner.grads[bp]
    _check(gw, rgw, torch.float32, acc_w, f"{name}: weight gradient")
    _check(gb, rgb, torch.float32, acc_b, f"{name}: bias gradient")
    if need_gx:
        # pad modes fold the padded gradient back: at most 2 copies per axis -> 8 more additions per element
        depth = co * kt * kh * kw + (8 if mode != "constant" else 0)
        acc_x = _gamma(depth, C_OF[gx_by]) * ax
        _check(gx.permute(0, 4, 1, 2, 3), rgx, torch.float32, acc_x, f"{name}: data gradient")
    else:
        assert gx is None
    if pad_[0] > 0:
        _, wgw, _ = _conv64_grads(x64, w64, b64, g64, *args[:3], mode, back=True)
        _rejects(gw, wgw, torch.float32, acc_w, f"{name}: time pad at the back")
    if kind == "ff":
        _, wgw, _ = _conv64_grads(video64[:, :, 1:2], w64, b64, g64, *args)
        _rejects(gw, wgw, torch.float32, acc_w, f"{name}: first-frame gradient taken from frame 1")


# ------------------------------------------------------------------------------------------------------------------
# C. every dgrad call of real training steps
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def dgrad_log(monkeypatch):
    """Records every TapeRunner._dgrad / DiscrRunner._dgrad_s2 call (copies of g, the weight and the result, the other
    arguments, the kernel that ran) and the runners that made them."""
    calls, runners = [], []

    def recording(fn, op):
        def wrapped(self, g, w, *args):
            if not any(r is self for r in runners):
                runners.append(self)
            kind, out = _launch(self.eng, lambda: fn(self, g, w, *args))
            calls.append(dict(op=op, g=g.detach().clone(), w=w.detach().clone(), args=args, out=out.clone(), kernel=kind))
            return out
        return wrapped

    monkeypatch.setattr(TapeRunner, "_dgrad", recording(TapeRunner._dgrad, "dgrad"))
    monkeypatch.setattr(DiscrRunner, "_dgrad_s2", recording(DiscrRunner._dgrad_s2, "s2"))
    return calls, runners


def _check_calls(calls):
    """Every recorded call against its float64 reference, with the Part A bound.  No call is cropped."""
    for i, c in enumerate(calls):
        g, out, what = c["g"], c["out"], f"call {i} ({c['op']}, {c['kernel']}, g {tuple(c['g'].shape)})"
        if c["op"] == "dgrad":
            k, out_spatial = c["args"][0], tuple(c["args"][1])
            ref, absr = _dgrad64(g, c["w"], k, out_spatial), _dgrad64(g.abs(), c["w"].abs(), k, out_spatial)
            K = c["w"].shape[0] * math.prod(k)
        else:      # dgrad weights (4 Ci, Co, 1, 1) of either builder == the 2x2 stride-2 forward weight, transposed
            wd = c["w"]
            w = wd[:, :, 0, 0].t().reshape(wd.shape[1], wd.shape[0], 1, 1)
            hw = tuple(c["args"][0][2:4])
            ref, absr = _s2_grad64(g, w, False, hw), _s2_grad64(g.abs(), w.abs(), False, hw)
            K = wd.shape[1]
        _check(out, ref, out.dtype, _gamma(K, C_OF[c["kernel"]]) * absr, what)
        del ref, absr


def _residual_units(m):
    n = 0
    for stages, layers in ((m.stages, m.encoder_layers), (list(reversed(m.stages)), m.decoder_layers)):
        for st, mod in zip(stages, layers):
            if st.kind == "residual":
                n += len(list(mod)) if st.nested else 1
    return n


@pytest.mark.parametrize("dt", ["bf16", "f32"])
def test_readme_generator_step_dgrad_calls(dgrad_log, dt):
    """One generator step of the README config (B = 1, 17 x 128 x 128; channels 64-512, frames 20 / 10 / 5, 128^2 down to
    16^2): every dgrad call against float64, and as many calls as the stages imply (two per ResidualUnit, plus conv_out with
    constant padding)."""
    calls, runners = dgrad_log
    dtype = DT[dt]
    gold = load_golden("readme")
    kw = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    assert kw == dict(gold["kwargs"])
    # the generator step without the GAN / perceptual terms, as the *_train goldens
    m = build_product(dict(kw, use_gan=False, perceptual_loss_weight=0., quantizer_aux_loss_weight=0.), gold["wseed"])
    m = m.cuda().to(dtype)
    m.train()
    total, _ = m(golden_video(gold).cuda().to(dtype), return_loss=True)
    total.backward()
    torch.cuda.synchronize()
    assert m.conv_out.pad_mode == "constant" and not m.separate_first_frame_encoding
    assert len(calls) == 2 * _residual_units(m) + 1
    assert len(runners) == 1 and runners[0].own_dgrad_calls == len(calls)
    conv_out = [c for c in calls if c["w"].shape[0] == 3]
    assert len(conv_out) == 1 and conv_out[0]["kernel"] == "simt"
    if dtype == torch.bfloat16:
        slab = {c["w"].shape[0] for c in calls if c["kernel"] == "slab" and c["args"][0] == K333}
        assert {64, 128, 256, 512} <= slab, slab
    else:
        assert all(c["kernel"] == "simt" for c in calls)
    del m, total
    _check_calls(calls)


def _discr_dgrad_calls(runner):
    """dgrad calls one DiscrRunner backward makes: per block the 3x3 net[2] conv and the unshuffle conv (if it
    down-samples), net[0] and conv_res unless it is the first block without an image gradient; the to_logits 3x3 conv."""
    n = 1
    for i, (block, _) in enumerate(runner.d.blocks):
        n += 1 + (block.downsample is not None)
        if i > 0 or runner.need_image_grad:
            n += 2
    return n


def test_mini_gan_discriminator_step_dgrad_calls(dgrad_log):
    """One bf16 discriminator step (return_discr_loss, no gradient penalty) of the mini_gan golden's config."""
    import synth_data
    calls, runners = dgrad_log
    gold = load_golden("mini_gan")
    torch.manual_seed(0)
    m = VideoTokenizer(**gold["kwargs"])
    synth_data.fill_state_dict_(m, gold["wseed"])
    synth_data.fill_discr_(m, gold["wseed"])
    m = m.cuda().bfloat16()
    m.train()
    torch.manual_seed(gold["step_seed"])
    total, _ = m(golden_video(gold).cuda().bfloat16(), return_discr_loss=True, apply_gradient_penalty=False)
    total.backward()
    torch.cuda.synchronize()
    assert runners and all(isinstance(r, DiscrRunner) for r in runners)
    assert len(calls) == sum(_discr_dgrad_calls(r) for r in runners) == sum(r.own_dgrad_calls for r in runners)
    kinds = {(c["op"], c["kernel"]) for c in calls}
    assert {("dgrad", "slab"), ("s2", "slab")} <= kinds, kinds
    del m, total
    _check_calls(calls)
