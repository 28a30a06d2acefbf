"""The perceptual loss of the generator step (reference M:1788-1810) on the device: a user-supplied VGG feature extractor
(``VideoTokenizer(vgg=<module>)``, M:1081, M:1397-1405) run on the engine's kernels, with the data gradient the adaptive
adversarial weight (M:1812-1841) and the tokenizer's backward need.

Accepted modules have torchvision's VGG layout (vgg11/13/16/19 without batch norm, classifier full or truncated):
``features`` = Conv2d(k=3, s=1, p=1) each followed by ReLU, and MaxPool2d(2, 2) after a ReLU; ``avgpool`` =
AdaptiveAvgPool2d; ``classifier`` = a Linear first, then Linear / ReLU / Dropout in any order.  torchvision is not
imported.

Division of labour
  * FORWARD: every 3x3 conv is an engine conv with ReLU in its epilogue, each 2x2 max-pool one ``mv2_maxpool2x2``.  The
    3-channel first conv takes conv_in's kw-packed ingest in bf16, as the discriminator's does.  The adaptive average
    pool is linear, so it is folded into the first Linear (``fold_avgpool_linear``), which then runs as a conv whose
    kernel covers the last feature map; later Linears are 1x1 convs.  ``channels == 1`` (the reference repeats the
    frame 3 times, M:1797-1799) sums the first conv's input-channel axis; ``channels == 4`` (the reference drops the 4th
    channel, M:1801-1803) gives it zero weights.  Neither copies the frames.
  * BACKWARD: the data gradient only -- the VGG is a frozen feature extractor no optimizer sees, so its parameters get no
    gradient (the reference's autograd would fill their ``.grad``; nothing reads it).  3x3 convs: TapeRunner._dgrad;
    pools: ``mv2_maxpool2x2_backward``, which applies the ReLU mask of the pooled conv; the other ReLU masks: an
    elementwise mask on the saved output; Linears: their transposed weights as 1x1 convs on the engine's kernels.
  * Dropout follows ``vgg.training`` as in the reference (the VGG is a submodule, so ``model.train()`` turns it on).  Its
    masks are drawn from torch's CUDA generator, so ``torch.manual_seed`` reproduces a step, and the backward reuses them.

The weight packs depend on the frame size (the average-pool fold) and are kept in a cache the tokenizer owns, keyed on
the VGG's parameters like the discriminator's packs: they do not survive ``deepcopy`` or pickling.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from ._lib import ACT_NONE, ACT_RELU
from .engine import PackCache, pack_conv, pack_conv_in_kwpack
from .train import TapeRunner


# --------------------------------------------------------------------------------------------
# structure check
# --------------------------------------------------------------------------------------------
def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def check_vgg(vgg):
    """Raises NotImplementedError naming the first child outside the layout the device path runs (module docstring)."""
    for name in ("features", "avgpool", "classifier"):
        if not isinstance(getattr(vgg, name, None), nn.Module):
            raise NotImplementedError(f"vgg: torchvision's VGG layout (features, avgpool, classifier) is required; no `{name}`")
    for name in ("features", "classifier"):
        if not isinstance(getattr(vgg, name), nn.Sequential):
            raise NotImplementedError(f"vgg.{name} must be an nn.Sequential, got {type(getattr(vgg, name)).__name__}")
    if not isinstance(vgg.avgpool, nn.AdaptiveAvgPool2d):
        raise NotImplementedError(f"vgg.avgpool: {vgg.avgpool!r} is not supported (AdaptiveAvgPool2d only)")
    feats = list(vgg.features.named_children())
    for name, m in feats:                          # unsupported types first (e.g. the BatchNorm2d of vgg*_bn) ...
        if not isinstance(m, (nn.Conv2d, nn.ReLU, nn.MaxPool2d)):
            raise NotImplementedError(f"vgg.features.{name}: {m!r} is not supported (Conv2d, ReLU and MaxPool2d only)")
    for i, (name, m) in enumerate(feats):          # ... then their parameters and order
        prev = feats[i - 1][1] if i > 0 else None
        nxt = feats[i + 1][1] if i + 1 < len(feats) else None
        if isinstance(m, nn.Conv2d):
            ok = (_pair(m.kernel_size) == (3, 3) and _pair(m.stride) == (1, 1) and _pair(m.padding) == (1, 1)
                  and _pair(m.dilation) == (1, 1) and m.groups == 1 and m.padding_mode == "zeros" and isinstance(nxt, nn.ReLU))
        elif isinstance(m, nn.ReLU):
            ok = isinstance(prev, nn.Conv2d)
        elif isinstance(m, nn.MaxPool2d):
            ok = (_pair(m.kernel_size) == (2, 2) and _pair(m.stride) == (2, 2) and _pair(m.padding) == (0, 0)
                  and _pair(m.dilation) == (1, 1) and not m.ceil_mode and not m.return_indices and isinstance(prev, nn.ReLU))
        else:
            ok = False
        if not ok:
            raise NotImplementedError(f"vgg.features.{name}: {m!r} is not supported (3x3 stride-1 pad-1 Conv2d + ReLU, "
                                      "MaxPool2d(2, 2) after a ReLU)")
    if not any(isinstance(m, nn.Conv2d) for _, m in feats):
        raise NotImplementedError("vgg.features has no Conv2d")
    if feats[0][1].in_channels != 3:
        raise NotImplementedError(f"vgg.features.{feats[0][0]}: the first conv must take 3 channels (RGB frames)")
    cls = list(vgg.classifier.named_children())
    for i, (name, m) in enumerate(cls):
        if not (isinstance(m, (nn.Linear, nn.ReLU, nn.Dropout)) and (i > 0 or isinstance(m, nn.Linear))):
            raise NotImplementedError(f"vgg.classifier.{name}: {m!r} is not supported (a Linear first, then Linear / ReLU / "
                                      "Dropout)")
    if not cls:
        raise NotImplementedError("vgg.classifier is empty (its first Linear absorbs the adaptive average pool)")


# --------------------------------------------------------------------------------------------
# host repacks (checked against torch's formulation on CPU, tests/test_vgg_cpu.py)
# --------------------------------------------------------------------------------------------
def _out_size(avgpool, fmap):
    os_ = _pair(avgpool.output_size)
    return tuple(fmap[i] if os_[i] is None else int(os_[i]) for i in range(2))


def adaptive_pool_matrix(n_in, n_out):
    """(n_out, n_in) float64: AdaptiveAvgPool's window i covers [floor(i n_in / n_out), ceil((i + 1) n_in / n_out))."""
    a = torch.zeros((n_out, n_in), dtype=torch.float64)
    for i in range(n_out):
        s, e = (i * n_in) // n_out, -(-((i + 1) * n_in) // n_out)
        a[i, s:e] = 1. / (e - s)
    return a


def fold_avgpool_linear(weight, channels, fmap, out_size):
    """Linear(C * oh * ow -> O) over the '(c h w)' flatten of AdaptiveAvgPool2d((oh, ow)) of a (C, h, w) map == a conv
    (O, C, h, w) covering the map: the pool's averaging matrices folded into the weights (fp32; folded in fp64)."""
    O = weight.shape[0]
    oh, ow = out_size
    w4 = weight.detach().double().reshape(O, channels, oh, ow)
    ah, aw = adaptive_pool_matrix(fmap[0], oh).to(w4.device), adaptive_pool_matrix(fmap[1], ow).to(w4.device)
    return torch.einsum("ocij,iy,jx->ocyx", w4, ah, aw).float()


def first_conv_weight(w, channels):
    """The first conv's weights for `channels`-channel frames: 1 -> the input-channel axis summed (the reference's repeat
    to 3 channels, M:1797-1799); 4 -> a zero 4th input channel (its slice to 3, M:1801-1803); 3 -> unchanged."""
    w = w.detach()
    if channels == 1:
        return w.float().sum(dim=1, keepdim=True)
    if channels == 4:
        return torch.cat((w, w.new_zeros((w.shape[0], 1) + tuple(w.shape[2:]))), dim=1)
    return w


def vgg_packs(vgg, eng, fmap_in, channels):
    """The weight packs of the VGG on engine eng for `channels`-channel frames of size fmap_in."""
    dt = eng.dtype
    feats = []                                     # {"pk", "w", "pool", ["kw"]} per conv
    h, w = fmap_in
    for m in vgg.features:
        if isinstance(m, nn.Conv2d):
            wt = first_conv_weight(m.weight, channels) if not feats else m.weight.detach()
            e = dict(pk=pack_conv(wt, m.bias, dt), w=wt, pool=False)
            if not feats and dt == torch.bfloat16 and wt.shape[1] * 3 <= 32:    # 3-channel first conv: kw-packed ingest
                e["kw"] = pack_conv_in_kwpack(wt[:, :, None], m.bias)
            feats.append(e)
        elif isinstance(m, nn.MaxPool2d):
            feats[-1]["pool"] = True
            h, w = h // 2, w // 2
    c_last = feats[-1]["w"].shape[0]
    ops = []
    for m in vgg.classifier:
        if isinstance(m, nn.Linear):
            if not ops:              # the first Linear with the average pool folded in: a conv covering the (h, w) map
                wf = fold_avgpool_linear(m.weight, c_last, (h, w), _out_size(vgg.avgpool, (h, w)))
                pk = pack_conv(wf, m.bias, dt)
                # its data gradient: a 1x1 conv O -> (h w c), whose output is the channels-last map gradient
                pk_t = pack_conv(wf.permute(2, 3, 1, 0).reshape(h * w * c_last, -1)[:, :, None, None], None, dt)
            else:
                pk = pack_conv(m.weight[:, :, None, None], m.bias, dt)
                pk_t = pack_conv(m.weight.detach().t()[:, :, None, None], None, dt)
            ops.append(dict(kind="linear", pk=pk, pk_t=pk_t))
        elif isinstance(m, nn.ReLU):
            ops.append(dict(kind="relu"))
        else:
            ops.append(dict(kind="dropout", mod=m))
    return dict(feats=feats, ops=ops, fmap=(h, w), c_last=c_last)


# --------------------------------------------------------------------------------------------
# torch restatement (channels-first): the CPU checks and the dropout test
# --------------------------------------------------------------------------------------------
def vgg_torch(vgg, x, masks=None):
    """vgg(x) of the accepted layout in torch ops: (B, 3, H, W) -> (B, features).  `masks`: one entry per classifier Dropout,
    the scaled keep-mask to multiply by (as VggRunner.masks records) or None for an inactive dropout; masks=None runs
    every Dropout as in eval()."""
    h = x
    for m in vgg.features:
        if isinstance(m, nn.Conv2d):
            h = F.conv2d(h, m.weight, m.bias, padding=1)
        elif isinstance(m, nn.ReLU):
            h = F.relu(h)
        else:
            h = F.max_pool2d(h, 2, 2)
    h = F.adaptive_avg_pool2d(h, _out_size(vgg.avgpool, h.shape[-2:])).flatten(1)
    k = 0
    for m in vgg.classifier:
        if isinstance(m, nn.Linear):
            h = F.linear(h, m.weight, m.bias)
        elif isinstance(m, nn.ReLU):
            h = F.relu(h)
        else:
            if masks is not None and masks[k] is not None:
                h = h * masks[k].to(h.device, h.dtype)
            k += 1
    return h


# --------------------------------------------------------------------------------------------
# device path
# --------------------------------------------------------------------------------------------
def _relu_grad(g, y):
    """d ReLU(x) / dx from the OUTPUT y (torch's threshold_backward): g where y > 0, else 0."""
    return torch.where(y > 0, g, torch.zeros_like(g))


class VggRunner(TapeRunner):
    """One VGG forward through the engine's kernels on (B, channels, H, W) frames, recording its data gradient."""

    def __init__(self, vgg, fmap_in, channels=3, cache=None):
        """`cache`: the PackCache the VGG's packs are kept in (None: packs of this runner's own)."""
        eng, self.P = (cache or PackCache()).get(vgg, "the VGG", lambda eng: vgg_packs(vgg, eng, fmap_in, channels),
                                                 key=(tuple(fmap_in), int(channels)))
        super().__init__(eng)
        self.vgg = vgg
        self.masks = []          # per classifier Dropout: the scaled keep-mask drawn, or None when inactive

    def forward(self, images, record=True):
        """images (B, channels, H, W) -> features (B, F) in the compute dtype.  record=False keeps no tape (the real frames)."""
        eng, P = self.eng, self.P
        imgs = images.detach().to(eng.dtype).contiguous()
        B = imgs.shape[0]
        x = None
        for i, e in enumerate(P["feats"]):
            if i == 0 and "kw" in e:
                pin = e["kw"]
                y = eng.conv(eng.ingest_kwpack(imgs[:, :, None], 0, pin), pin, pad=(0, 1, 0), act=ACT_RELU)
            else:
                if i == 0:
                    x = eng.to_channels_last(imgs[:, :, None])
                y = eng.conv(x, e["pk"], act=ACT_RELU)
            out = eng.maxpool2x2(y) if e["pool"] else y
            if record:
                def bwd(g, e=e, y=y):
                    gz = eng.maxpool2x2_backward(g, y) if e["pool"] else _relu_grad(g, y)
                    return self._dgrad(gz, e["w"], (1, 3, 3), y.shape[1:4])
                self.tape.append(bwd)
            x = out
        h, w = P["fmap"]
        ops = P["ops"]
        skip = False
        for j, op in enumerate(ops):
            if skip:                               # a ReLU fused into the Linear before it
                skip = False
                continue
            if op["kind"] == "linear":
                fuse = j + 1 < len(ops) and ops[j + 1]["kind"] == "relu"
                act = ACT_RELU if fuse else ACT_NONE
                xin = x
                if j == 0:
                    y = eng.conv(x, op["pk"], pad=(0, 0, 0), out_spatial=(1, 1, 1), act=act)
                else:
                    y = eng.conv(x, op["pk"], act=act)
                skip = fuse
                if record:
                    def bwd(g, op=op, y=y, fuse=fuse, shape=tuple(xin.shape)):
                        if fuse:
                            g = _relu_grad(g, y)
                        return eng.conv(g.contiguous(), op["pk_t"]).reshape(shape)
                    self.tape.append(bwd)
            elif op["kind"] == "relu":
                y = torch.relu(x)
                if record:
                    self.tape.append(lambda g, y=y: _relu_grad(g, y))
            else:
                m = op["mod"]
                mask = None
                if self.vgg.training and m.p > 0:
                    mask = torch.empty_like(x).bernoulli_(1. - m.p).div_(1. - m.p)
                    y = x * mask
                else:
                    y = x
                self.masks.append(mask)
                if record and mask is not None:
                    self.tape.append(lambda g, mask=mask: g * mask)
            x = y
        return x.reshape(B, -1)

    def backward(self, g_feats):
        """g_feats (B, F) -> the data gradient wrt the images (B, channels, H, W).  Single use: the tape is released."""
        g = self._run_tape(g_feats.to(self.eng.dtype).reshape(g_feats.shape[0], 1, 1, 1, -1),
                           "the VGG's backward ran already, or its forward kept no tape")
        return g[:, 0].permute(0, 3, 1, 2).contiguous()


class _PerceptualFn(torch.autograd.Function):
    """(real frames, recon frames) -> F.mse_loss(vgg(real), vgg(recon)) (M:1805-1808).  The gradient wrt the recon frames
    is computed in the forward (the adaptive weight needs it before the total backward); the backward scales it."""

    @staticmethod
    def forward(ctx, vgg, channels, cache, out, real, fake):
        fmap = tuple(fake.shape[-2:])
        ra = VggRunner(vgg, fmap, channels, cache)
        f_real = ra.forward(real, record=False)                   # the reference's order: real first, then recon (M:1805-1806)
        rb = VggRunner(vgg, fmap, channels, cache)
        f_fake = rb.forward(fake, record=out["need_grad"])
        out["masks"] = (ra.masks, rb.masks)
        loss = rb.eng.mse(f_real, f_fake).to(fake.dtype)
        ctx.gx = None
        if out["need_grad"]:
            g = (f_fake.float() - f_real.float()) * (2. / f_fake.numel())
            ctx.gx = rb.backward(g)
            out["grad_frames"] = ctx.gx
        return loss

    @staticmethod
    def backward(ctx, g):
        gx = None if ctx.gx is None else ctx.gx * g.to(ctx.gx.dtype)
        return None, None, None, None, None, gx


def perceptual_loss(vgg, real, fake, channels=3, cache=None):
    """F.mse_loss(vgg(real), vgg(fake)) of (B, channels, H, W) frames on the device, differentiable wrt `fake` (first
    order).  -> (loss 0-d in fake's dtype, info): info["grad_frames"] is d loss / d fake (present when a gradient is
    needed), info["masks"] the dropout masks drawn for (real, fake)."""
    if fake.device.type != "cuda" or real.device != fake.device:
        raise RuntimeError(f"the perceptual loss runs on CUDA: frames on {real.device} / {fake.device}")
    if real.shape != fake.shape or real.ndim != 4 or real.shape[1] != channels:
        raise ValueError(f"frames must both be (B, {channels}, H, W), got {tuple(real.shape)} / {tuple(fake.shape)}")
    w0 = vgg.features[0].weight
    if w0.device != fake.device:
        raise RuntimeError(f"frames are on {fake.device} but the VGG is on {w0.device}")
    info = dict(need_grad=torch.is_grad_enabled() and fake.requires_grad)
    with torch.cuda.device(fake.device):
        loss = _PerceptualFn.apply(vgg, channels, cache, info, real, fake)
    return loss, info
