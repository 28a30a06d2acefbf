"""The image discriminator of the GAN loss (reference M:549-675) on the device, and the loss terms built on it
(``return_discr_loss``, M:1731-1786; the adversarial generator term, M:1826-1843, ``generator_term``: its image gradient is
computed in the forward, so that the adaptive adversarial weight can use it before the total backward).

Division of labour (as in train.py)
  * FORWARD: the engine's sm_90a kernels.  Every 3x3 conv carries LeakyReLU(0.1) in its epilogue; the block output
    ``(downsample(net(x)) + conv_res(x)) * 2^-0.5`` is one conv with the scaled-residual epilogue (epi_mode 2).  The
    pixel-unshuffle + 1x1 ``downsample`` is repacked once as a 2x2 stride-2 conv (no rearranged copy), ``conv_res`` is a
    1x1 stride-2 conv, the 3-channel first conv takes conv_in's kw-packed ingest (bf16), and the Linear of ``to_logits``
    is a conv whose kernel covers the whole last feature map, with its weights read in channels-last order.  The
    attention blocks run through Engine.linear_attention / Engine.feed_forward with T = 1.
  * BACKWARD: data gradients of the 3x3 convs and of both stride-2 convs on the engine's conv kernels (the dgrad of the
    2x2/s2 conv is a 1x1 conv with the depth-to-space store; the 1x1/s2 conv is its one-phase case); weight / bias
    gradients through ``aten.convolution_backward``; the attention blocks through their torch restatements (train.py).
  * GRADIENT PENALTY (M:102-115): a double backward, computed with torch autograd (``create_graph=True``) on the torch
    restatement ``discriminator_torch`` re-evaluated from the saved frames.  This is library code that runs only on
    penalty steps and carries no speed claim.

The discriminator's weight packs live on the Discriminator itself, keyed on its own parameters: a discriminator optimizer
step leaves the generator's packs and CUDA graphs alone, and a generator step leaves the discriminator's.
"""
from __future__ import annotations

from collections import namedtuple

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from ._lib import ACT_LEAKY_RELU, ACT_NONE, SHUFFLE_SPACE
from .engine import pack_conv, pack_conv_in_kwpack, pack_feed_forward, pack_linear_attention
from .train import TapeRunner, _feed_forward_block, _linear_attention_block

# reference M:1039-1043
DiscrLossBreakdown = namedtuple("DiscrLossBreakdown", ["discr_loss", "multiscale_discr_losses", "gradient_penalty"])

_RES_SCALE = 2 ** -0.5


# --------------------------------------------------------------------------------------------
# host repacks (each is checked against the reference's formulation on CPU, tests/test_gan_cpu.py)
# --------------------------------------------------------------------------------------------
def unshuffle_conv_weight(w):
    """'b c (h p1) (w p2) -> b (c p1 p2) h w' followed by a 1x1 conv (Co, 4 C, 1, 1) == a 2x2 stride-2 conv (Co, C, 2, 2)."""
    return w.reshape(w.shape[0], w.shape[1] // 4, 2, 2)


def unshuffle_dgrad_weight(w):
    """Data gradient of the 2x2 stride-2 conv: a 1x1 conv C_out -> 4 C_in whose output rows are in the '(c p1 p2)' order of
    the depth-to-space store: (4 Ci, Co, 1, 1)."""
    return w.reshape(w.shape[0], -1).t()[:, :, None, None]


def stride2_1x1_dgrad_weight(w):
    """Data gradient of a 1x1 stride-2 conv (Co, Ci, 1, 1): the one-phase case of the above -- only the p1 = p2 = 0
    rows of the depth-to-space output are non-zero."""
    Co, Ci = w.shape[:2]
    wd = w.new_zeros((Ci, 4, Co))
    wd[:, 0] = w.reshape(Co, Ci).t()
    return wd.reshape(4 * Ci, Co)[:, :, None, None]


def logits_conv_weight(lin, dim_last, fmap):
    """Linear(latent -> 1) over the '(c h w)' flatten (M:664-665) == a conv (1, C, h, w) covering the whole last feature map;
    the conv pack reads it in channels-last order."""
    return lin.weight.reshape(1, dim_last, fmap[0], fmap[1])


# --------------------------------------------------------------------------------------------
# torch restatement (channels-first): the gradient penalty's double backward and the CPU checks
# --------------------------------------------------------------------------------------------
def discriminator_torch(d, x):
    """Discriminator.forward (M:669-675) in torch: (B, C, H, W) -> logits (B,)."""
    for block, attn in d.blocks:
        cr = block.conv_res
        res = F.conv2d(x, cr.weight, cr.bias, stride=cr.stride)
        h = F.leaky_relu(F.conv2d(x, block.net[0].weight, block.net[0].bias, padding=1), 0.1)
        h = F.leaky_relu(F.conv2d(h, block.net[2].weight, block.net[2].bias, padding=1), 0.1)
        if block.downsample is not None:
            ds = block.downsample[1]
            h = F.conv2d(F.pixel_unshuffle(h, 2), ds.weight, ds.bias)
        x = (h + res) * _RES_SCALE
        xl = x.permute(0, 2, 3, 1)[:, None]
        xl = _linear_attention_block(xl, attn[0].fn)
        xl = _feed_forward_block(xl, attn[1].fn, False)
        x = xl[:, 0].permute(0, 3, 1, 2)
    tl = d.to_logits
    h = F.leaky_relu(F.conv2d(x, tl[0].weight, tl[0].bias, padding=1), 0.1)
    return F.linear(h.flatten(1), tl[3].weight, tl[3].bias)[:, 0]


def gradient_penalty(d, images):
    """M:102-115 on the torch restatement: ((|d logits.sum() / d images|_2 per sample) ** 2).mean(), differentiable wrt
    the discriminator's parameters."""
    x = images.detach().requires_grad_(True)
    with torch.enable_grad():
        out = discriminator_torch(d, x)
        g, = torch.autograd.grad(out, x, torch.ones_like(out), create_graph=True)
        return (g.reshape(g.shape[0], -1).norm(2, dim=1) ** 2).mean()


# --------------------------------------------------------------------------------------------
# device path
# --------------------------------------------------------------------------------------------
def _packs(d, eng):
    """The weight packs of the Discriminator d on engine eng."""
    dt = eng.dtype
    P = []
    for block, attn in d.blocks:
        n0, n2, cr = block.net[0], block.net[2], block.conv_res
        e = dict(net0=pack_conv(n0.weight, n0.bias, dt), net2=pack_conv(n2.weight, n2.bias, dt),
                 res=pack_conv(cr.weight, cr.bias, dt), attn=pack_linear_attention(attn[0].fn, dt),
                 ff=pack_feed_forward(attn[1].fn, dt))
        if dt == torch.bfloat16 and n0.weight.shape[1] * 3 <= 32:       # 3-channel first conv: conv_in's kw-packed ingest
            e["net0_kw"] = pack_conv_in_kwpack(n0.weight[:, :, None], n0.bias)
        # the block output (branch + conv_res(x)) * 2^-0.5 is the epilogue of the block's last conv: the unshuffle conv
        # with conv_res(x) as residual, or -- without downsample -- conv_res with the branch as residual
        if block.downsample is not None:
            ds = block.downsample[1]
            e["down"] = pack_conv(unshuffle_conv_weight(ds.weight), ds.bias, dt)
            e["down"].epi_mode = 2
        else:
            e["res"].epi_mode = 2
        P.append(e)
    tl = d.to_logits
    logits = dict(conv=pack_conv(tl[0].weight, tl[0].bias, dt),
                  lin=pack_conv(logits_conv_weight(tl[3], tl[0].weight.shape[0], d.last_fmap), tl[3].bias, dt))
    return P, logits


def _leaky_grad(g, y):
    """d LeakyReLU(x) / dx from the OUTPUT y (leaky ReLU preserves sign): 1 for y > 0, 0.1 otherwise."""
    return g * torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.1))


class DiscrRunner(TapeRunner):
    """One discriminator forward through the engine's kernels, recording what the backward needs."""

    def __init__(self, d):
        eng, (self.P, self.logits_pk) = d._pack_cache.get(d, "the discriminator", lambda eng: _packs(d, eng))
        super().__init__(eng)
        self.d = d

    def _dgrad_s2(self, g, wd, x_shape):
        """Data gradient of a stride-2 conv whose dgrad weights `wd` (4 Ci, Co, 1, 1) feed the depth-to-space store."""
        eng = self.eng
        gx = eng.conv(g.contiguous(), pack_conv(wd, None, eng.dtype, shuffle_q=4), shuffle=SHUFFLE_SPACE)
        assert tuple(gx.shape) == tuple(x_shape), (gx.shape, x_shape)
        self.own_dgrad_calls += 1
        return gx

    def _block(self, x, e, block, first, images):
        eng = self.eng
        B, _, H, W, _ = x.shape
        n0, n2, cr = block.net[0], block.net[2], block.conv_res
        if "net0_kw" in e:
            pin = e["net0_kw"]
            h1 = eng.conv(eng.ingest_kwpack(images[:, :, None], 0, pin), pin, pad=(0, 1, 0), act=ACT_LEAKY_RELU)
        else:
            h1 = eng.conv(x, e["net0"], act=ACT_LEAKY_RELU)
        down = block.downsample is not None
        if down:
            Ho, Wo = H // 2, W // 2
            res = eng.conv(x, e["res"], stride=(1, 2, 2), pad=(0, 0, 0), out_spatial=(1, Ho, Wo))
            h2 = eng.conv(h1, e["net2"], act=ACT_LEAKY_RELU)
            out = eng.conv(h2, e["down"], stride=(1, 2, 2), pad=(0, 0, 0), out_spatial=(1, Ho, Wo), res=res)
        else:
            h2 = eng.conv(h1, e["net2"], act=ACT_LEAKY_RELU)
            out = eng.conv(x, e["res"], res=h2)

        need_gx = not first or self.need_image_grad

        def bwd(g):
            g = g * _RES_SCALE                     # d out / d (branch) for both branches
            res_stride = (1, 2, 2) if down else (1, 1, 1)
            if down:
                ds = block.downsample[1]          # pixel-unshuffle + 1x1 conv as the 2x2 stride-2 conv (unshuffle_conv_weight)
                self._wgrad(g, h2.permute(0, 4, 1, 2, 3), ds.weight, ds.bias, (1, 2, 2), (1, 2, 2), (0, 0, 0))
                gz2 = _leaky_grad(self._dgrad_s2(g, unshuffle_dgrad_weight(ds.weight.detach()), h2.shape), h2)
            else:
                gz2 = _leaky_grad(g, h2)
            gh1 = self._conv_bwd(gz2, h1, n2.weight, n2.bias, (1, 3, 3))
            gz1 = _leaky_grad(gh1, h1)
            if first:
                v = images.to(eng.dtype)
                # the first block's input is the images (channels-first): weight gradients on them, data gradients optional
                self._conv_bwd(gz1, v[:, :, None], n0.weight, n0.bias, (1, 3, 3), pad=(0, 1, 1), need_gx=False, x_is_cf=True)
                self._wgrad(g, x.permute(0, 4, 1, 2, 3), cr.weight, cr.bias, (1, 1, 1), res_stride, (0, 0, 0))
                if not need_gx:
                    return None
                gx = self._dgrad(gz1, n0.weight, (1, 3, 3), x.shape[1:4])
            else:
                gx = self._conv_bwd(gz1, x, n0.weight, n0.bias, (1, 3, 3))
                self._wgrad(g, x.permute(0, 4, 1, 2, 3), cr.weight, cr.bias, (1, 1, 1), res_stride, (0, 0, 0))
            if down:
                return gx + self._dgrad_s2(g, stride2_1x1_dgrad_weight(cr.weight.detach()), x.shape)
            return gx + self._dgrad(g, cr.weight, (1, 1, 1), x.shape[1:4])

        self.tape.append(bwd)
        return out

    def forward(self, images, need_image_grad=False):
        """images (B, C, H, W) -> logits (B,) in the compute dtype."""
        eng, d = self.eng, self.d
        self.need_image_grad = need_image_grad
        imgs = images.detach().to(eng.dtype).contiguous()
        x = eng.to_channels_last(imgs[:, :, None])
        for i, ((block, attn), e) in enumerate(zip(d.blocks, self.P)):
            x = self._block(x, e, block, i == 0, imgs)
            la, ff = attn[0].fn, attn[1].fn
            xa = x
            x = eng.linear_attention(xa, e["attn"])
            self.tape.append(lambda g, xa=xa, la=la: self._vjp(lambda t: _linear_attention_block(t, la), xa, list(la.parameters()), g))
            xf = x
            x = eng.feed_forward(xf, e["ff"])
            self.tape.append(lambda g, xf=xf, ff=ff: self._vjp(lambda t: _feed_forward_block(t, ff, False), xf,
                                                                list(ff.parameters()), g))
        tl = d.to_logits
        xl = x
        h = eng.conv(xl, self.logits_pk["conv"], act=ACT_LEAKY_RELU)
        logits = eng.conv(h, self.logits_pk["lin"], pad=(0, 0, 0), out_spatial=(1, 1, 1), act=ACT_NONE)

        def bwd_logits(g):       # g: (B,) -> gradient wrt the last feature map (channels-last)
            lin = tl[3]          # the Linear as the conv covering the last feature map (logits_conv_weight)
            g5 = g.reshape(-1, 1, 1, 1, 1).to(h.dtype)
            gh = self._wgrad(g5, h.permute(0, 4, 1, 2, 3), lin.weight, lin.bias, (1,) + tuple(d.last_fmap), (1, 1, 1), (0, 0, 0),
                             need_gx=True)
            gz = _leaky_grad(gh.permute(0, 2, 3, 4, 1).contiguous(), h)
            return self._conv_bwd(gz, xl, tl[0].weight, tl[0].bias, (1, 3, 3))

        self.tape.append(bwd_logits)
        return logits.reshape(-1)

    def backward(self, g_logits):
        """-> (gradient wrt the images (B, C, H, W) | None, {Parameter: grad})."""
        g = self._run_tape(g_logits.to(self.eng.dtype),
                           "the discriminator's backward ran already (retain_graph is not supported by this path)")
        gx = None if g is None else g[:, 0].permute(0, 3, 1, 2).contiguous()
        return gx, self.grads


class _DiscriminatorFn(torch.autograd.Function):
    """(images, *parameters) -> logits: forward by the engine kernels, backward by DiscrRunner's tape (first order only)."""

    @staticmethod
    def forward(ctx, runner, images, *params):
        logits = runner.forward(images, need_image_grad=ctx.needs_input_grad[1])
        ctx.runner, ctx.params = runner, params
        return logits

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        gx, grads = ctx.runner.backward(g)
        return (None, gx) + tuple(grads[p] if p in grads else torch.zeros_like(p) for p in ctx.params)


class _GeneratorTermFn(torch.autograd.Function):
    """(images, *parameters) -> hinge_gen_loss = -logits.mean() (M:123-124).  When a gradient is needed, the tape runs in
    the forward: the image gradient is then available to the adaptive adversarial weight (M:1837) before the total
    backward, and the backward only scales it and the discriminator's parameter gradients by grad_out."""

    @staticmethod
    def forward(ctx, runner, info, images, *params):
        logits = runner.forward(images, need_image_grad=info["image_grad"])
        loss = -logits.mean()
        ctx.gx, ctx.grads, ctx.params = None, None, params
        if info["need_grad"]:
            gx, grads = runner.backward(torch.full_like(logits, -1. / logits.numel()))
            ctx.gx, ctx.grads = gx, [grads.get(p) for p in params]
            info["grad_images"] = gx
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        gx = None if ctx.gx is None else ctx.gx * g.to(ctx.gx.dtype)
        return (None, None, gx) + tuple(torch.zeros_like(p) if gp is None else gp * g.to(gp.dtype)
                                        for p, gp in zip(ctx.params, ctx.grads))


def _check_images(d, images):
    if images.ndim != 4 or images.shape[1] != d.channels or tuple(images.shape[-2:]) != tuple(d.image_size):
        raise ValueError(f"images must be (B, {d.channels}, {d.image_size[0]}, {d.image_size[1]}), got {tuple(images.shape)}")
    w0 = d.to_logits[0].weight
    if images.device != w0.device:
        raise RuntimeError(f"images are on {images.device} but the discriminator is on {w0.device}")
    return w0.device


def discriminator_forward(d, images):
    """Discriminator(images): (B, C, H, W) on the device -> logits (B,) in the model dtype, differentiable (first order)
    wrt the images and every discriminator parameter."""
    dev = _check_images(d, images)
    runner = DiscrRunner(d)
    with torch.cuda.device(dev):
        return _DiscriminatorFn.apply(runner, images, *[p for p in d.parameters()])


def generator_term(d, images):
    """The adversarial generator term -discr(images).mean() (M:1826-1831) -> (loss 0-d, info): differentiable (first order)
    wrt the images and every discriminator parameter, like -discriminator_forward(d, images).mean(); info["grad_images"] is
    d loss / d images, present when the images need a gradient."""
    dev = _check_images(d, images)
    params = list(d.parameters())
    info = dict(image_grad=images.requires_grad,
                need_grad=torch.is_grad_enabled() and (images.requires_grad or any(p.requires_grad for p in params)))
    runner = DiscrRunner(d)
    with torch.cuda.device(dev):
        return _GeneratorTermFn.apply(runner, info, images, *params), info
