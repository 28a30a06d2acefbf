"""Parameter containers of the H100 VideoTokenizer.

These ``nn.Module`` classes hold parameters under exactly the attribute paths of the reference
model so that ``state_dict()`` keys are interchangeable with reference checkpoints
(SURVEY.md 8b; reference key layout e.g. ``encoder_layers.2.0.fn.0.conv.weight``).  They do NOT
compute: the forward path is executed by ``engine.Engine`` through the C ABI, which reads the
parameters.  Calling ``forward`` on a container is an error (there is no eager fallback).

Reference construction sites are cited per class (M: = magvit2_pytorch/magvit2_pytorch.py).
"""
from __future__ import annotations

import math

import torch
from torch import nn

from ._lib import SHUFFLE_NONE, SHUFFLE_TIME
from .engine import PackCache, pack_conv, tf32_matmul_enabled


class _NoForward(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(
            f"{type(self).__name__} is a parameter container; the forward path runs through "
            "libmagvit2_b200.so (VideoTokenizer.tokenize / decode_from_code_indices / forward)")


class Marker(_NoForward):
    """Parameter-free placeholder keeping nn.Sequential indices aligned with the reference
    (ELU / LeakyReLU / Sigmoid / SiLU / Rearrange slots)."""

    def __init__(self, what: str):
        super().__init__()
        self.what = what

    def extra_repr(self):
        return self.what


class CausalConv3d(_NoForward):
    """M:892-928 -- weights live in ``.conv`` (an nn.Conv3d used purely as storage)."""

    def __init__(self, chan_in, chan_out, kernel_size, pad_mode="constant"):
        super().__init__()
        ks = kernel_size if isinstance(kernel_size, tuple) else (kernel_size,) * 3
        assert ks[1] % 2 == 1 and ks[2] % 2 == 1
        self.kernel_size = tuple(ks)
        self.pad_mode = pad_mode
        self.conv = nn.Conv3d(chan_in, chan_out, ks)


class SqueezeExcite(_NoForward):
    """M:194-219 -- to_k: C->1, net: C->max(16, C//2)->C; last conv zero weight, bias -10."""

    def __init__(self, dim, dim_hidden_min=16, init_bias=-10.):
        super().__init__()
        hidden = max(dim_hidden_min, dim // 2)
        self.to_k = nn.Conv2d(dim, 1, 1)
        self.net = nn.Sequential(nn.Conv2d(dim, hidden, 1), Marker("LeakyReLU(0.1)"),
                                 nn.Conv2d(hidden, dim, 1), Marker("Sigmoid"))
        nn.init.zeros_(self.net[2].weight)
        nn.init.constant_(self.net[2].bias, init_bias)


class Residual(_NoForward):
    """M:167-174."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class TokenShift(_NoForward):
    """M:244-254."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn


def residual_unit(dim, kernel_size):
    """M:930-944: Residual(Sequential(CausalConv3d, ELU, Conv3d 1x1x1, ELU, SqueezeExcite))."""
    return Residual(nn.Sequential(
        CausalConv3d(dim, dim, kernel_size), Marker("ELU"),
        nn.Conv3d(dim, dim, 1), Marker("ELU"),
        SqueezeExcite(dim)))


class Conv3DMod(_NoForward):
    """M:680-716 -- StyleGAN2-style modulated causal conv: one ``weights`` Parameter (dim_out, dim, kt, ks, ks), demod=True."""

    def __init__(self, dim, spatial_kernel, time_kernel, eps=1e-8):
        super().__init__()
        self.eps = eps
        self.spatial_kernel, self.time_kernel = spatial_kernel, time_kernel
        self.weights = nn.Parameter(torch.randn((dim, dim, time_kernel, spatial_kernel, spatial_kernel)))
        nn.init.kaiming_normal_(self.weights, a=0, mode="fan_in", nonlinearity="selu")


class ResidualUnitMod(_NoForward):
    """M:946-976 -- to_cond: Linear(dim_cond -> dim), conv: Conv3DMod, conv_out: Conv3d 1x1x1 (no SqueezeExcite)."""

    def __init__(self, dim, kernel_size, dim_cond):
        super().__init__()
        ks = kernel_size if isinstance(kernel_size, tuple) else (kernel_size,) * 3
        assert ks[1] == ks[2]
        self.to_cond = nn.Linear(dim_cond, dim)
        self.conv = Conv3DMod(dim, spatial_kernel=ks[1], time_kernel=ks[0])
        self.conv_out = nn.Conv3d(dim, dim, 1)


class SpatialDownsample2x(_NoForward):
    """M:757-768 (antialias=False)."""

    def __init__(self, dim, dim_out):
        super().__init__()
        self.conv = nn.Conv2d(dim, dim_out, 3, stride=2, padding=1)


class TimeDownsample2x(_NoForward):
    """M:782-794."""

    def __init__(self, dim, dim_out):
        super().__init__()
        self.conv = nn.Conv1d(dim, dim_out, 3, stride=2)


def _repeat_init_(conv, factor):
    # M:829-836 / M:866-873: kaiming-uniform a (o/factor) kernel and repeat it `factor` times
    w = conv.weight
    base = torch.empty(w.shape[0] // factor, *w.shape[1:])
    nn.init.kaiming_uniform_(base)
    with torch.no_grad():
        w.copy_(base.repeat_interleave(factor, dim=0))
        conv.bias.zero_()


class SpatialUpsample2x(_NoForward):
    """M:811-836: net = (Conv2d dim->4*dim_out 1x1, SiLU, depth-to-space)."""

    def __init__(self, dim, dim_out):
        super().__init__()
        conv = nn.Conv2d(dim, dim_out * 4, 1)
        self.net = nn.Sequential(conv, Marker("SiLU"), Marker("depth_to_space 2x2"))
        _repeat_init_(conv, 4)


class TimeUpsample2x(_NoForward):
    """M:848-873: net = (Conv1d dim->2*dim_out k1, SiLU, depth-to-time)."""

    def __init__(self, dim, dim_out):
        super().__init__()
        conv = nn.Conv1d(dim, dim_out * 2, 1)
        self.net = nn.Sequential(conv, Marker("SiLU"), Marker("depth_to_time x2"))
        _repeat_init_(conv, 2)


class RMSNorm(_NoForward):
    """M:258-273: gamma is (C,) channel-last or (C,1,1,1) channel-first ((C,1,1) for images)."""

    def __init__(self, dim, channel_first=False, images=False):
        super().__init__()
        self.channel_first = channel_first
        self.gamma = nn.Parameter(torch.ones(((dim, 1, 1) if images else (dim, 1, 1, 1)) if channel_first else (dim,)))


class Attention(_NoForward):
    """M:327-368 (Space/TimeAttention share the parameter layout, M:444-464)."""

    def __init__(self, dim, dim_head, heads, causal, num_memory_kv=4):
        super().__init__()
        inner = dim_head * heads
        self.dim, self.dim_head, self.heads, self.causal = dim, dim_head, heads, causal
        self.norm = RMSNorm(dim)
        self.to_qkv = nn.Sequential(nn.Linear(dim, inner * 3, bias=False), Marker("split qkv heads"))
        self.mem_kv = nn.Parameter(torch.randn(2, heads, num_memory_kv, dim_head))
        self.to_out = nn.Sequential(Marker("merge heads"), nn.Linear(inner, dim, bias=False))


class TaylorSeriesLinearAttn(_NoForward):
    """Parameter layout of the un-vendored dependency (SURVEY.md Appendix A.3)."""

    def __init__(self, dim, dim_head, heads):
        super().__init__()
        inner = dim_head * heads
        self.to_q = nn.Sequential(nn.Linear(dim, inner, bias=False), Marker("split heads"))
        self.to_kv = nn.Sequential(nn.Linear(dim, inner * 2, bias=False), Marker("split kv heads"))
        self.to_out = nn.Sequential(nn.Linear(inner, dim, bias=False), Marker("Dropout(0)"))


class LinearSpaceAttention(_NoForward):
    """M:390-442."""

    def __init__(self, dim, dim_head, heads):
        super().__init__()
        self.dim, self.dim_head, self.heads = dim, dim_head, heads
        self.norm = RMSNorm(dim)
        self.attn = TaylorSeriesLinearAttn(dim, dim_head, heads)


class SimpleGateLoopLayer(_NoForward):
    """Parameter layout of gateloop_transformer.SimpleGateLoopLayer(dim) with its defaults (prenorm RMSNorm, no post-LN), as
    the reference constructs it at M:1220-1221: ``norm.gamma`` (dim,), ``to_qkva.0.weight`` (3 dim, dim), no bias."""

    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.norm = RMSNorm(dim)
        self.to_qkva = nn.Sequential(nn.Linear(dim, dim * 3, bias=False), Marker("'b n (qkva d) -> qkva (b d) n 1'"))


class ToTimeSequence(_NoForward):
    """M:178-191."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class FeedForward(_NoForward):
    """M:471-496: channel-first RMSNorm, Conv3d C->2I 1x1x1, GEGLU, Conv3d I->C; I = int(C*4*2/3).
    images=True (the discriminator's blocks): Conv2d and a (C, 1, 1) gamma."""

    def __init__(self, dim, mult=4, images=False):
        super().__init__()
        inner = int(dim * mult * 2 / 3)
        self.dim, self.dim_inner = dim, inner
        self.norm = RMSNorm(dim, channel_first=True, images=images)
        conv = nn.Conv2d if images else nn.Conv3d
        self.net = nn.Sequential(conv(dim, inner * 2, 1), Marker("GEGLU"), conv(inner, dim, 1))


class DiscriminatorBlock(_NoForward):
    """M:549-586 (antialiased_downsample=False): conv_res 1x1 (stride 2 when downsampling), net = 3x3 conv, LeakyReLU,
    3x3 conv, LeakyReLU, downsample = pixel-unshuffle + 1x1 conv; output (downsample(net(x)) + conv_res(x)) * 2^-0.5."""

    def __init__(self, input_channels, filters, downsample=True):
        super().__init__()
        self.conv_res = nn.Conv2d(input_channels, filters, 1, stride=(2 if downsample else 1))
        self.net = nn.Sequential(nn.Conv2d(input_channels, filters, 3, padding=1), Marker("LeakyReLU(0.1)"),
                                 nn.Conv2d(filters, filters, 3, padding=1), Marker("LeakyReLU(0.1)"))
        self.downsample = nn.Sequential(Marker("'b c (h p1) (w p2) -> b (c p1 p2) h w'"),
                                        nn.Conv2d(filters * 4, filters, 1)) if downsample else None


class Discriminator(_NoForward):
    """M:588-675: the image discriminator of the GAN loss.  Parameters only -- ``VideoTokenizer.discr`` runs it on the
    device (gan.py).  Blur (antialiased_downsample) needs kornia's filter3d and is not supported; the linear attention
    kernel takes dim_head 8 only."""

    def __init__(self, *, dim, image_size, channels=3, max_dim=512, attn_heads=8, attn_dim_head=32, linear_attn_dim_head=8,
                 linear_attn_heads=16, ff_mult=4, antialiased_downsample=False):
        super().__init__()
        if antialiased_downsample:
            raise NotImplementedError("Discriminator(antialiased_downsample=True): Blur needs kornia's filter3d, which is "
                                      "not supported")
        if linear_attn_dim_head != 8:
            raise NotImplementedError("Discriminator: the linear attention kernel takes linear_attn_dim_head = 8 only")
        hw = tuple(image_size) if isinstance(image_size, (tuple, list)) else (image_size, image_size)
        num_layers = int(math.log2(min(hw)) - 2)
        layer_dims = [channels] + [(dim * 4) * (2 ** i) for i in range(num_layers + 1)]
        layer_dims = [min(d, max_dim) for d in layer_dims]
        dims_in_out = list(zip(layer_dims[:-1], layer_dims[1:]))
        self.image_size, self.channels = hw, channels
        self.blocks = nn.ModuleList([])
        for ind, (cin, cout) in enumerate(dims_in_out):
            block = DiscriminatorBlock(cin, cout, downsample=ind != len(dims_in_out) - 1)
            attn = nn.Sequential(Residual(LinearSpaceAttention(cout, linear_attn_dim_head, linear_attn_heads)),
                                 Residual(FeedForward(cout, mult=ff_mult, images=True)))
            self.blocks.append(nn.ModuleList([block, attn]))
        dim_last = layer_dims[-1]
        self.last_fmap = tuple(n // 2 ** num_layers for n in hw)
        latent = self.last_fmap[0] * self.last_fmap[1] * dim_last
        self.to_logits = nn.Sequential(nn.Conv2d(dim_last, dim_last, 3, padding=1), Marker("LeakyReLU(0.1)"),
                                       Marker("'b ... -> b (...)'"), nn.Linear(latent, 1), Marker("'b 1 -> b'"))
        self._pack_cache = PackCache()       # engine and weight packs of the device path (gan.py)

    def forward(self, images):
        from .gan import discriminator_forward
        return discriminator_forward(self, images)


class LFQ(_NoForward):
    """Parameter/buffer layout of vector_quantize_pytorch.LFQ (SURVEY.md Appendix A.1):
    persistent int64 ``mask``, Linear ``project_in`` / ``project_out`` (with bias) between ``dim`` and
    ``log2(codebook_size) * num_codebooks`` channels."""

    def __init__(self, dim, codebook_size, entropy_loss_weight, commitment_loss_weight, diversity_gamma,
                 soft_clamp_input_value, num_codebooks=1, spherical=False):
        super().__init__()
        d = int(math.log2(codebook_size))
        assert 2 ** d == codebook_size, "codebook_size must be a power of two"
        self.dim, self.codebook_size, self.codebook_dim = dim, codebook_size, d
        self.num_codebooks = int(num_codebooks)
        self.spherical = bool(spherical)
        self.entropy_loss_weight = entropy_loss_weight
        self.commitment_loss_weight = commitment_loss_weight
        self.diversity_gamma = diversity_gamma
        self.soft_clamp_input_value = soft_clamp_input_value
        cdims = d * self.num_codebooks
        if dim == cdims:
            raise NotImplementedError("LFQ without projections (dim == log2(codebook_size) * num_codebooks) is not supported")
        if cdims > 32:
            raise NotImplementedError("the quantiser kernels take at most 32 projected dims (log2(codebook_size) * num_codebooks)")
        self.project_in = nn.Linear(dim, cdims)
        self.project_out = nn.Linear(cdims, dim)
        self.register_buffer("mask", 2 ** torch.arange(d - 1, -1, -1))


class FSQ(_NoForward):
    """Parameter layout of vector_quantize_pytorch.FSQ (SURVEY.md Appendix A.2)."""

    def __init__(self, levels, dim, num_codebooks=1):
        super().__init__()
        self.levels = [int(l) for l in levels]
        self.num_codebooks = int(num_codebooks)
        self.dim, self.codebook_dim = dim, len(levels)
        self.codebook_size = int(math.prod(self.levels))
        cdims = len(levels) * self.num_codebooks
        if dim == cdims:
            raise NotImplementedError("FSQ without projections is not supported")
        if cdims > 32:
            raise NotImplementedError("the quantiser kernels take at most 32 projected dims (len(levels) * num_codebooks)")
        self.project_in = nn.Linear(dim, cdims)
        self.project_out = nn.Linear(cdims, dim)


class CausalConvTranspose3d(nn.Module):
    """M:990-1024 -- ``nn.ConvTranspose3d`` with stride (time_stride, 1, 1), padding (0, kh//2, kw//2), output cut to
    ``t * time_stride`` frames.  The reference never instantiates it inside ``VideoTokenizer`` (dead code there); it is kept
    as a standalone, *computing* module for API completeness (SURVEY.md 8f N4).

    On the device a transposed conv with time stride s is s causal convs interleaved in time:
        out[s t' + r] = sum_m  x[t' - m] * W[:, :, r + m s]        (spatially: a stride-1 conv with the flipped kernel)
    so it runs as ONE causal conv with s * C_out output channels in the reference's '(c p)' order and ceil(kt / s) taps,
    followed by the depth-to-time store the TimeUpsample2x kernels already have (time_stride 1 or 2)."""

    def __init__(self, chan_in, chan_out, kernel_size, *, time_stride, **kwargs):
        super().__init__()
        ks = kernel_size if isinstance(kernel_size, tuple) else (kernel_size,) * 3
        assert ks[1] % 2 == 1 and ks[2] % 2 == 1
        if time_stride not in (1, 2):
            raise NotImplementedError("CausalConvTranspose3d on the device supports time_stride 1 and 2")
        self.upsample_factor = time_stride
        self.conv = nn.ConvTranspose3d(chan_in, chan_out, ks, (time_stride, 1, 1), padding=(0, ks[1] // 2, ks[2] // 2), **kwargs)
        self._pack_cache = PackCache()

    def equivalent_conv_weight(self):
        """-> (weight (s*Co, Ci, ceil(kt/s), kh, kw), bias (s*Co) | None) of the causal conv described above."""
        w = self.conv.weight.detach()                      # (Ci, Co, kt, kh, kw)
        s = self.upsample_factor
        Ci, Co, kt, kh, kw = w.shape
        ktp = -(-kt // s)
        wf = w.flip(3, 4).permute(1, 0, 2, 3, 4)           # (Co, Ci, kt, kh, kw), spatially flipped
        weq = w.new_zeros((Co, s, Ci, ktp, kh, kw))
        for r in range(s):
            for dt in range(ktp):
                j = r + (ktp - 1 - dt) * s
                if j < kt:
                    weq[:, r, :, dt] = wf[:, :, j]
        beq = None if self.conv.bias is None else self.conv.bias.detach().repeat_interleave(s)
        return weq.reshape(Co * s, Ci, ktp, kh, kw), beq

    def forward(self, x):
        assert x.ndim == 5
        w = self.conv.weight
        if w.device.type != "cuda" or x.device != w.device:
            raise RuntimeError("CausalConvTranspose3d runs on CUDA (sm_90a) only, input and parameters on the same device")
        with torch.no_grad(), torch.cuda.device(w.device):
            # an fp32 pack carries the CUDA-core and the TF32 layouts; the call runs TF32 while torch allows TF32 matmuls
            eng, pk = self._pack_cache.get(self, "CausalConvTranspose3d", lambda eng: pack_conv(
                *self.equivalent_conv_weight(), eng.dtype, shuffle_q=self.upsample_factor,
                tc=True if eng.dtype == torch.float32 else None), half=True)
            eng.tf32 = w.dtype == torch.float32 and tf32_matmul_enabled()
            y = eng.conv(eng.to_channels_last(x), pk, shuffle=SHUFFLE_TIME if self.upsample_factor == 2 else SHUFFLE_NONE)
            out = eng.to_channels_first(y)
            n = self.output_frames(x.shape[2])
            return out if n == out.shape[2] else out[:, :, :n].contiguous()

    def output_frames(self, t: int) -> int:
        """min(t * s, (t - 1) * s + kt): a kernel shorter than the stride leaves the transposed conv's output shorter than the cut."""
        s, kt = self.upsample_factor, self.conv.weight.shape[2]
        return min(t * s, (t - 1) * s + kt)
