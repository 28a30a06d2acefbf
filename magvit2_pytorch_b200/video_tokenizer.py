"""H100-native drop-in for the reference ``VideoTokenizer`` inference path.

Mirrors the reference class's public surface (magvit2_pytorch/magvit2_pytorch.py:1045-1720 =
M:): the keyword-only constructor and ``layers=(...)`` spec (M:1047-1092, M:1138-1318),
``tokenize`` (M:1651), ``decode_from_code_indices`` (M:1579), ``forward`` inference returns
(M:1657-1720), ``encode`` / ``decode`` (M:1523, M:1598), ``parameters()`` as a list (M:1460),
``state_dict`` key layout (SURVEY.md 8b), ``save`` / ``load`` / ``init_and_load_from``
(M:1447-1458, M:1495-1520), ``copy_for_eval`` (M:1476), ``device`` (M:1443).

All arithmetic runs in hand-written sm_90a kernels behind the C ABI of libmagvit2_b200.so;
the compute dtype follows the parameters' dtype (``.float()`` -> fp32 CUDA-core path, or the same wgmma kernels in TF32
for calls without gradients while torch allows TF32 matmuls, ``.bfloat16()`` -> bf16 wgmma path, ``.half()`` -> the same
wgmma kernels in fp16: no-grad calls only, no discriminator / VGG).  There is no CPU / eager fallback.

``cond_residual`` layers (ResidualUnitMod / Conv3DMod, M:680-753, M:946-988) run on the device through the
factorisation in include/magvit2_b200.h; the other ``cond_*`` types raise in the reference itself.
``separate_first_frame_encoding`` (M:1113-1120, M:1553-1561, M:1633-1639) runs through the same conv kernels.
``forward(return_loss=True)`` (reconstruction + quantiser auxiliary loss; models built with ``use_gan=False,
perceptual_loss_weight=0``) runs on the device; in ``model.train()`` with gradients enabled it returns a loss with a
``grad_fn`` (train.py: forward by the same kernels, backward by library code).
Models that use the GAN (``use_gan=True, adversarial_loss_weight > 0``) build the image discriminator ``discr``
(M:1415-1422) and run it on the device (gan.py): ``return_discr_loss`` (M:1731-1786) and the adversarial generator term of
``return_loss`` (M:1826-1843).  The perceptual term (``perceptual_loss_weight > 0``, ``channels`` in {1, 3, 4}) needs a
user-supplied VGG module (``vgg=``, M:1081; nothing is downloaded): the perceptual loss and the adaptive adversarial weight
(M:1788-1841) then run on the device (vgg.py).  Without one (``vgg=None``) the model builds no discriminator and
``return_loss`` / ``return_discr_loss`` raise.  The VGG is left out of ``state_dict``, ``copy_for_eval`` and the pickled
config, so ``init_and_load_from`` gives a model without it.
``encode``, ``decode`` and ``decode_from_code_indices`` are differentiable like the reference's (M:1522-1649) when grad
mode is on and a floating input requires grad or, in train mode, a parameter the call reaches does (_grad_params): the
forward runs on the same kernels and train.py's tape pieces give the gradients of the video / latents, ``cond`` and the
reached parameters; every other call takes the no-grad path unchanged.  ``tokenize`` stays no-grad, as in the reference.
``attn_dropout`` (0 <= p < 1) drops the softmax attention weights of train-mode forwards (grad and no-grad) with a Philox
mask seeded once per call from torch's default CPU generator (engine.AttnDropout, DESIGN.md 3.6); such forwards bypass the
CUDA graphs.  Eval mode never drops.
Multiscale discriminators (``multiscale_discrs=``, M:1085, M:1429-1441) are the user's own torch modules on whole videos and
torch runs them, as in the reference: ``return_discr_loss`` adds their hinge losses on the video and the detached
reconstruction (M:1752-1765).  The generator term reproduces the reference's quirk (M:1846-1866): its loop never calls the
discriminators -- each multiscale generator loss is ``-frames.mean()`` of the image-GAN term's picked reconstruction frames
(the perceptual term's without an image GAN), and its adaptive weight, with a VGG, is the perceptual gradient norm over that
loss's (clamped at 1e-5, no NaN fallback).  They are left out of ``parameters()``, ``discr_parameters()``, ``copy_for_eval``
and the pickled config (the reference trainer builds their optimizers itself), and kept in ``state_dict``.
Out of scope (raise at construction; SURVEY.md 8f): the discriminator's antialiased (Blur) downsampling.
"""
from __future__ import annotations

import contextlib
import copy
import functools
import pickle
from collections import namedtuple
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import modules as M
from .engine import AttnDropout, Engine, PackCache, tf32_matmul_enabled

__version__ = "0.1.0"


# reference M:1028-1037
LossBreakdown = namedtuple("LossBreakdown", [
    "recon_loss", "lfq_aux_loss", "quantizer_loss_breakdown", "perceptual_loss", "adversarial_gen_loss",
    "adaptive_adversarial_weight", "multiscale_gen_losses", "multiscale_gen_adaptive_weights"])


def _hinge_discr_loss(fake, real):
    """hinge_discr_loss (M:120-121)."""
    return (F.relu(1 + fake) + F.relu(1 - real)).mean()


@dataclass
class Stage:
    kind: str          # residual | compress_space | compress_time | attend_space | linear_attend_space | attend_time
    dim: int
    dim_out: int
    count: int = 1
    nested: bool = False


def _on_model_device(fn):
    """Runs the method with the model's CUDA device current: the C ABI launches on the current device (kernels, TMA
    descriptors, function attributes), so a tokenizer on cuda:1 must not be driven while cuda:0 is current."""
    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        dev = self.device
        ctx = torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()
        with ctx:
            return fn(self, *a, **k)
    return wrapper


def _attn_dropout_scope(fn):
    """Runs the method with attention dropout live when the model is in training mode and was built with attn_dropout > 0:
    one 64-bit Philox seed per call, drawn from torch's default CPU generator (torch.manual_seed reproduces a step and nothing
    waits on the device; nothing is drawn otherwise, so other runs' random streams are untouched)."""
    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        if not (self.training and self.attn_dropout > 0.):
            return fn(self, *a, **k)
        eng = self.engine
        if eng.dropout is not None:           # already inside a dropout forward of this model
            return fn(self, *a, **k)
        hi, lo = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
        eng.dropout = AttnDropout(self.attn_dropout, hi << 32 | lo)
        try:
            return fn(self, *a, **k)
        finally:
            eng.dropout = None
    return wrapper


def _precision_scope(fn):
    """Runs the method with the engine's fp32 precision at IEEE unless the method turns TF32 on (VideoTokenizer._tf32_engine),
    and restores the caller's afterwards: a call that takes gradients, or a nested call, never inherits TF32."""
    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        eng = self._engine
        prev = False if eng is None else eng.tf32
        if eng is not None:
            eng.tf32 = False
        try:
            return fn(self, *a, **k)
        finally:
            if self._engine is not None:
                self._engine.tf32 = prev
    return wrapper


_UNSUPPORTED_LAYERS = {
    "cond_attend_space": "raises in the reference itself (SURVEY.md 2 row 9)",
    "cond_linear_attend_space": "raises in the reference itself (SURVEY.md 2 row 9)",
    "cond_attend_time": "raises in the reference itself (SURVEY.md 2 row 9)",
}


class VideoTokenizer(nn.Module):
    def __init__(
        self,
        *,
        image_size,
        layers: Tuple = ("residual", "residual", "residual"),
        residual_conv_kernel_size=3,
        num_codebooks=1,
        codebook_size: Optional[int] = None,
        channels=3,
        init_dim=64,
        max_dim=float("inf"),
        dim_cond=None,
        dim_cond_expansion_factor=4.,
        input_conv_kernel_size: Tuple[int, int, int] = (7, 7, 7),
        output_conv_kernel_size: Tuple[int, int, int] = (3, 3, 3),
        pad_mode: str = "constant",
        lfq_entropy_loss_weight=0.1,
        lfq_commitment_loss_weight=1.,
        lfq_diversity_gamma=2.5,
        lfq_spherical=False,
        quantizer_aux_loss_weight=1.,
        lfq_soft_clamp_input_value=10.,
        lfq_activation=None,
        use_fsq=False,
        fsq_levels: Optional[List[int]] = None,
        attn_dim_head=32,
        attn_heads=8,
        attn_dropout=0.,
        linear_attn_dim_head=8,
        linear_attn_heads=16,
        vgg=None,
        vgg_weights=None,
        perceptual_loss_weight=1e-1,
        discr_kwargs: Optional[dict] = None,
        multiscale_discrs: Tuple = tuple(),
        use_gan=True,
        adversarial_loss_weight=1.,
        grad_penalty_loss_weight=10.,
        multiscale_adversarial_loss_weight=1.,
        flash_attn=True,
        separate_first_frame_encoding=False,
    ):
        super().__init__()
        cfg = dict(locals())
        cfg.pop("self")
        cfg.pop("__class__", None)
        for k in ("vgg", "lfq_activation"):      # modules are not part of the pickled config here
            cfg[k] = None
        cfg["multiscale_discrs"] = tuple()
        self._configs = pickle.dumps(cfg)       # M:1097-1100

        if not isinstance(layers, tuple):
            raise TypeError("layers must be a tuple")
        if pad_mode not in ("constant", "reflect", "replicate", "circular"):
            raise ValueError(f"unknown pad_mode {pad_mode!r}")
        if not 0. <= attn_dropout <= 1.:                                          # as nn.Dropout (A:175)
            raise ValueError(f"dropout probability has to be between 0 and 1, but got {attn_dropout}")
        if attn_dropout == 1.:
            raise NotImplementedError("attn_dropout=1 would drop every attention weight; it is not supported")
        self.attn_dropout = float(attn_dropout)
        ks = residual_conv_kernel_size

        self.channels = channels
        self.image_size = image_size
        self.conv_in = M.CausalConv3d(channels, init_dim, tuple(input_conv_kernel_size), pad_mode)
        self.conv_in_first_frame = nn.Identity()
        self.conv_out_first_frame = nn.Identity()
        self.separate_first_frame_encoding = bool(separate_first_frame_encoding)
        if separate_first_frame_encoding:                                          # M:1113-1120: SameConv2d (M:887-890)
            ik, ok = tuple(input_conv_kernel_size)[-2:], tuple(output_conv_kernel_size)[-2:]
            self.conv_in_first_frame = nn.Conv2d(channels, init_dim, ik, padding=(ik[0] // 2, ik[1] // 2))
            self.conv_out_first_frame = nn.Conv2d(init_dim, channels, ok, padding=(ok[0] // 2, ok[1] // 2))
        self.encoder_layers = nn.ModuleList([])
        self.decoder_layers = nn.ModuleList([])
        self.conv_out = M.CausalConv3d(init_dim, channels, tuple(output_conv_kernel_size), pad_mode)

        # ---- layer schedule (M:1129-1318) ----
        dim = init_dim
        fmap = image_size
        tdf = 1
        has_cond = False
        stages: List[Stage] = []
        for layer_def in layers:
            kind, *params = layer_def if isinstance(layer_def, tuple) else (layer_def,)
            dim_out = dim
            if kind in _UNSUPPORTED_LAYERS:
                raise NotImplementedError(f"layer type {kind!r}: {_UNSUPPORTED_LAYERS[kind]}")
            if has_cond and kind != "cond_residual":
                # has_cond is never reset in the reference (M:1153, M:1318): every later layer is called with cond=, and its
                # plain layers then raise TypeError -- only specs whose conditioned layers are the trailing ones run there
                raise TypeError(f"layer {kind!r} after a cond_* layer: the reference passes cond= to it and fails (M:1153, M:1318)")
            if kind == "residual":
                enc, dec = M.residual_unit(dim, ks), M.residual_unit(dim, ks)
                stages.append(Stage("residual", dim, dim, 1, False))
            elif kind == "cond_residual":                                        # M:1150-1157
                assert dim_cond is not None, "dim_cond must be passed into VideoTokenizer, if tokenizer is to be conditioned"
                has_cond = True
                dc = int(dim_cond * dim_cond_expansion_factor)
                enc, dec = M.ResidualUnitMod(dim, ks, dc), M.ResidualUnitMod(dim, ks, dc)
                stages.append(Stage("cond_residual", dim, dim))
            elif kind == "consecutive_residual":
                n, = params
                enc = nn.Sequential(*[M.residual_unit(dim, ks) for _ in range(n)])
                dec = nn.Sequential(*[M.residual_unit(dim, ks) for _ in range(n)])
                stages.append(Stage("residual", dim, dim, int(n), True))
            elif kind == "compress_space":
                dim_out = params[0] if len(params) > 0 else dim * 2
                dim_out = int(min(dim_out, max_dim))
                enc, dec = M.SpatialDownsample2x(dim, dim_out), M.SpatialUpsample2x(dim_out, dim)
                assert fmap > 1
                fmap //= 2
                stages.append(Stage(kind, dim, dim_out))
            elif kind == "compress_time":
                dim_out = params[0] if len(params) > 0 else dim * 2
                dim_out = int(min(dim_out, max_dim))
                enc, dec = M.TimeDownsample2x(dim, dim_out), M.TimeUpsample2x(dim_out, dim)
                tdf *= 2
                stages.append(Stage(kind, dim, dim_out))
            elif kind == "attend_space":
                def mk():
                    return nn.Sequential(M.Residual(M.Attention(dim, attn_dim_head, attn_heads, causal=False)),
                                         M.Residual(M.FeedForward(dim)))
                enc, dec = mk(), mk()
                stages.append(Stage(kind, dim, dim))
            elif kind == "linear_attend_space":
                def mk():
                    return nn.Sequential(M.Residual(M.LinearSpaceAttention(dim, linear_attn_dim_head, linear_attn_heads)),
                                         M.Residual(M.FeedForward(dim)))
                enc, dec = mk(), mk()
                stages.append(Stage(kind, dim, dim))
            elif kind == "gateloop_time":                                        # M:1216-1222
                enc = M.ToTimeSequence(M.Residual(M.SimpleGateLoopLayer(dim)))
                dec = M.ToTimeSequence(M.Residual(M.SimpleGateLoopLayer(dim)))
                stages.append(Stage(kind, dim, dim))
            elif kind == "attend_time":
                def mk():
                    return nn.Sequential(
                        M.Residual(M.TokenShift(M.Attention(dim, attn_dim_head, attn_heads, causal=True))),
                        M.Residual(M.TokenShift(M.FeedForward(dim))))
                enc, dec = mk(), mk()
                stages.append(Stage(kind, dim, dim))
            else:
                raise ValueError(f"unknown layer type {kind}")          # M:1311-1312
            self.encoder_layers.append(enc)
            self.decoder_layers.insert(0, dec)
            dim = dim_out

        # final LayerNorm: constructed and present in state_dict but never executed by the reference
        # (zip truncation at M:1565; SURVEY.md 3.1) -- kept for checkpoint compatibility only.
        self.encoder_layers.append(nn.Sequential(M.Marker("to channels-last"), nn.LayerNorm(dim), M.Marker("to channels-first")))

        self.stages = stages
        self.time_downsample_factor = tdf
        self.time_padding = tdf - 1
        self.fmap_size = fmap
        self.has_cond = has_cond
        self.has_cond_across_layers = [st.kind == "cond_residual" for st in stages]
        self.dim_cond = dim_cond
        self.encoder_cond_in = nn.Identity()
        self.decoder_cond_in = nn.Identity()
        if has_cond:                                                              # M:1340-1352: Linear + SiLU stems
            dc = int(dim_cond * dim_cond_expansion_factor)
            self.encoder_cond_in = nn.Sequential(nn.Linear(dim_cond, dc), M.Marker("SiLU"))
            self.decoder_cond_in = nn.Sequential(nn.Linear(dim_cond, dc), M.Marker("SiLU"))

        # ---- quantiser (M:1356-1384) ----
        self.use_fsq = use_fsq
        if not use_fsq:
            assert codebook_size is not None and fsq_levels is None, \
                "if use_fsq is set to False, `codebook_size` must be set (and not `fsq_levels`)"
            self.quantizers = M.LFQ(dim, codebook_size, lfq_entropy_loss_weight, lfq_commitment_loss_weight,
                                    lfq_diversity_gamma, lfq_soft_clamp_input_value, num_codebooks, lfq_spherical)   # M:1364-1373
        else:
            assert codebook_size is None and fsq_levels is not None, \
                "if use_fsq is set to True, `fsq_levels` must be set (and not `codebook_size`)"
            self.quantizers = M.FSQ(fsq_levels, dim, num_codebooks)                        # M:1378-1382
        self.quantizer_aux_loss_weight = quantizer_aux_loss_weight
        self.register_buffer("zero", torch.tensor(0.), persistent=False)

        # training-only branches of the reference.  The perceptual term runs when a VGG module is passed (vgg.py; this
        # package never downloads torchvision's weights, M:1397-1405); the image discriminator is built for the GAN term unless
        # the loss has a perceptual term without a VGG module (M:1415-1427, gan.py); the multiscale discriminators are the
        # user's modules, held even when the flags are off (M:1429-1441)
        self.vgg = None
        self.use_vgg = False
        self._vgg_cache = PackCache()           # the VGG's engine and weight packs (vgg.vgg_packs): per model, like _engine
        self.perceptual_loss_weight = perceptual_loss_weight
        if isinstance(vgg, nn.Module) and self._has_vgg():
            from .vgg import check_vgg
            check_vgg(vgg)
            self.vgg = vgg
            self.use_vgg = True
        self.use_gan = use_gan
        self.has_gan = False
        self.discr = None
        if use_gan and adversarial_loss_weight > 0. and (self.use_vgg or not self._has_vgg()):
            kw = dict(dim=dim, image_size=image_size, channels=channels, max_dim=512) if discr_kwargs is None else dict(discr_kwargs)
            self.discr = M.Discriminator(**kw)
            self.has_gan = True
        self.has_multiscale_gan = bool(use_gan and multiscale_adversarial_loss_weight > 0.)
        self.multiscale_discrs = nn.ModuleList([*multiscale_discrs])
        self.has_multiscale_discrs = bool(self.has_multiscale_gan and len(multiscale_discrs) > 0)
        self.adversarial_loss_weight = adversarial_loss_weight
        self.grad_penalty_loss_weight = grad_penalty_loss_weight
        self.multiscale_adversarial_loss_weight = multiscale_adversarial_loss_weight

        self.quantizer_loss_breakdown = None     # set by a train-mode forward (LFQ): (per_sample_entropy, batch_entropy, commitment)
        self.quantizer_aux_loss = None
        self._engine: Optional[Engine] = None
        # opt-in: replay each (entry point, input shape) as one CUDA graph after a warm-up call -- the forward path is
        # a static launch plan (~170 kernels), so this removes the per-launch host overhead.  Outputs are cloned out
        # of the graph's static buffers.
        self.cuda_graphs = False
        self._graphs = {}
        # graph-cache lane: calls issued under different lanes (host_io.StreamLanes: one CUDA stream per lane) replay
        # separate graph instances with their own static buffers and memory pools, so they may overlap on the device
        self._lane = 0
        # opt-in: programmatic dependent launch for every kernel of the path (mv2_set_pdl); process-wide library state
        self.pdl = False

    # ------------------------------------------------------------------ module plumbing
    @property
    def device(self):
        return self.zero.device

    def parameters(self, recurse: bool = True):
        # list, as the reference returns (M:1460-1471)
        return [*self.conv_in.parameters(), *self.conv_in_first_frame.parameters(), *self.conv_out_first_frame.parameters(),
                *self.conv_out.parameters(), *self.encoder_layers.parameters(),
                *self.decoder_layers.parameters(), *self.encoder_cond_in.parameters(), *self.decoder_cond_in.parameters(),
                *self.quantizers.parameters()]

    def discr_parameters(self):
        return [] if self.discr is None else list(self.discr.parameters())

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        # the VGG is left out of checkpoints, as the reference's remove_vgg does (M:141-155, M:1487-1489); filtering the
        # result keeps the module tree itself untouched
        if len(args) > 1:                       # torch's deprecated positional form (destination, prefix, keep_vars)
            prefix = args[1]
        sd = super().state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)
        for k in [k for k in sd if k.startswith(prefix + "vgg.")]:
            del sd[k]
        return sd

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        # reference checkpoints carry discriminator weights (always constructed, M:1422); a model that built no
        # discriminator drops them, and a model that holds no multiscale discriminators drops theirs (init_and_load_from builds
        # none).  Checkpoints carry no VGG weights (M:1491-1493): any in `state_dict` are ignored and the VGG keeps its own,
        # which stand in for its keys under strict loading.
        sd = {k: v for k, v in state_dict.items()
              if not ((self.discr is None and k.startswith("discr.")) or k.startswith("vgg.")
                      or (len(self.multiscale_discrs) == 0 and k.startswith("multiscale_discrs.")))}
        if self.vgg is not None:
            sd.update(("vgg." + k, v) for k, v in self.vgg.state_dict(keep_vars=True).items())
        return super().load_state_dict(sd, strict=strict, **kw)

    def __deepcopy__(self, memo):
        # the engine (packed weights, ctypes handles) and captured CUDA graphs (static buffers, private pools) belong
        # to THIS instance: a copy starts without them and re-packs / re-captures on first use
        eng, self._engine = self._engine, None
        graphs, self._graphs = self._graphs, {}
        try:
            cls = self.__class__
            new = cls.__new__(cls)
            memo[id(self)] = new
            for k, v in self.__dict__.items():
                new.__dict__[k] = copy.deepcopy(v, memo)
        finally:
            self._engine = eng
            self._graphs = graphs
        return new

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        st["_graphs"] = {}
        return st

    def copy_for_eval(self):
        """An eval-mode copy without the VGG and the multiscale discriminators (M:1476-1485): its return_loss raises like a
        model built with vgg=None, and has no multiscale terms."""
        dev = self.device
        memo = {id(self.multiscale_discrs): nn.ModuleList()}          # neither the multiscale discriminators ...
        if self.vgg is not None:
            memo[id(self.vgg)] = None                                 # ... nor the VGG is copied: the copy's `vgg` entry is None
        c = copy.deepcopy(self.cpu(), memo)
        self.to(dev)
        c.vgg, c.use_vgg = None, False
        c.has_multiscale_discrs = False
        c.eval()
        return c.to(dev)

    @classmethod
    def init_and_load_from(cls, path, strict=True):
        """M:1447-1458: a model built from the checkpoint's pickled config, which stores neither the VGG nor the multiscale
        discriminators: the model has neither, and the checkpoint's multiscale discriminator weights are dropped."""
        path = Path(path)
        assert path.exists()
        pkg = torch.load(str(path), map_location="cpu", weights_only=False)
        assert "config" in pkg, "model configs were not found in this saved checkpoint"
        config = pickle.loads(pkg["config"])
        # reference checkpoints pickle module-valued kwargs we do not build; the VGG is never saved, so a model loaded here
        # has none (vgg=None): pass the VGG module to the constructor and load_state_dict to train with the perceptual term;
        # likewise the multiscale discriminators
        for k in ("vgg", "lfq_activation"):
            config[k] = None
        config["multiscale_discrs"] = tuple()
        tok = cls(**config)
        tok.load(path, strict=strict)
        return tok

    def save(self, path, overwrite=True):
        path = Path(path)
        assert overwrite or not path.exists(), f"{str(path)} already exists"
        torch.save(dict(model_state_dict=self.state_dict(), version=__version__, config=self._configs), str(path))

    def load(self, path, strict=True):
        path = Path(path)
        assert path.exists()
        pkg = torch.load(str(path), map_location="cpu", weights_only=False)
        sd = pkg.get("model_state_dict")
        assert sd is not None
        self.load_state_dict(sd, strict=strict)

    # ------------------------------------------------------------------ engine access
    @property
    def engine(self) -> Engine:
        if self._engine is None:
            self._engine = Engine(self)
        self._engine.prepare()
        self._engine.lib.mv2_set_pdl(1 if self.pdl else 0)
        return self._engine

    def _tf32_engine(self, follow: bool = True) -> Engine:
        """The engine for a call without gradients, with an fp32 model's dense contractions on the TF32 tensor cores when
        `follow` and torch allows TF32 matmuls (tf32_matmul_enabled, read once here per call); bf16 / fp16 models are not
        affected.  Calls with gradients, and the discriminator and VGG, never come here: they stay IEEE fp32."""
        eng = self.engine
        eng.tf32 = bool(follow) and self.dtype == torch.float32 and tf32_matmul_enabled()
        if eng.tf32:
            eng.prepare()             # adds the TF32 packs on the first such call
        return eng

    def _graph_call(self, name, fn, *tensors):
        """fn(*tensors) -> tensor | tuple of tensors, replayed through a cached CUDA graph when enabled.  Forwards with live
        attention dropout run directly: a captured graph would replay one dropout mask forever."""
        if not self.cuda_graphs or (self._engine is not None and self._engine.dropout is not None):
            return fn(*tensors)
        eng = self.engine
        key = (name, eng._sig_id, tuple((tuple(t.shape), t.dtype) for t in tensors), self._lane, eng.tf32)
        if any(k[1] != eng._sig_id for k in self._graphs):      # parameters were re-packed: old graphs read stale weights
            self._graphs = {k: v for k, v in self._graphs.items() if k[1] == eng._sig_id}
        ent = self._graphs.get(key)
        if ent is None:                       # first call: plain run (warms up lazy init: attributes, entry points)
            self._graphs[key] = "warm"
            return fn(*tensors)
        if ent == "warm":                     # second call: capture
            static_in = [torch.empty_like(t) for t in tensors]
            for s_, t in zip(static_in, tensors):
                s_.copy_(t)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            l0 = eng.launches
            with torch.cuda.graph(g):
                out = fn(*static_in)
            ent = (g, static_in, out, eng.launches - l0)
            self._graphs[key] = ent
            g.replay()
        else:
            g, static_in, out, n_launch = ent
            for s_, t in zip(static_in, tensors):
                s_.copy_(t, non_blocking=True)
            g.replay()
            eng.launches += n_launch
        out = ent[2]
        if isinstance(out, tuple):
            return tuple(o.clone() for o in out)
        return out.clone()

    def _check_video(self, v, video_contains_first_frame=True):
        assert v.ndim in {4, 5}                                                   # M:1675
        assert tuple(v.shape[-2:]) == (self.image_size, self.image_size)          # M:1677
        if v.ndim == 4:                                                           # M:1681-1685
            v = v[:, :, None]
            video_contains_first_frame = True
        frames = v.shape[2]
        ff = int(bool(video_contains_first_frame))
        assert (frames - ff) % self.time_downsample_factor == 0, \
            f"number of frames {frames} minus the first frame ({frames - ff}) must be divisible by the total " \
            f"downsample factor across time {self.time_downsample_factor}"      # M:1691
        assert v.shape[1] == self.channels
        if v.device != self.device:
            raise RuntimeError(f"input is on {v.device} but the tokenizer is on {self.device}")
        return v, bool(ff)

    # ------------------------------------------------------------------ reference API
    def _grad_params(self, inputs, entry, *args):
        """The parameters handed to the differentiable path when encode / decode / decode_from_code_indices take it, else
        None.  The rule: grad mode is on, and a floating input requires grad or, in train mode, a parameter the call reaches
        does (the rule forward applies to return_loss).  Every other call runs the no-grad path (fused ResidualUnit, CUDA
        graphs, lanes).  entry, args: train.reached_parameters'."""
        if not torch.is_grad_enabled():
            return None
        wants_input = any(t is not None and t.is_floating_point() and t.requires_grad for t in inputs)
        if not (wants_input or self.training):
            return None
        from .train import reached_parameters
        params = reached_parameters(self, entry, *args)
        if not (wants_input or params):
            return None
        if self.dtype == torch.float16:
            raise TypeError(f"{entry} with gradients is not supported for float16 models (fp16 runs the no-grad path only): "
                            "call it under torch.no_grad() / in eval mode with inputs that do not require grad, or use "
                            "float32 / bfloat16 parameters")
        return params

    def _grad_call(self, method, x, cond, params, *args):
        """One differentiable call: train.TrainRunner.<method>(x, cond, *args) under train._TapeFn."""
        from .train import TrainRunner, _TapeFn
        runner = TrainRunner(self)
        run = getattr(runner, method)
        return _TapeFn.apply(runner, lambda x_, c_: run(x_, c_, *args), x, cond, *params), runner

    @_on_model_device
    @_precision_scope
    @_attn_dropout_scope
    def encode(self, video, quantize=False, cond=None, video_contains_first_frame=True):
        """M:1523-1576.  Returns (B, C, T', H', W') like the reference; quantize: (quantized, codes[, aux_loss]).
        Differentiable (see _grad_params) wrt the video, cond and the parameters it reaches (train.reached_parameters).  With
        quantize, LFQ passes a straight-through gradient in train mode only and FSQ in both modes; the third element keeps
        its no-grad value (zero in eval mode) -- the train-mode entropy loss with its gradient comes from forward(return_loss=True)."""
        video, ff = self._check_video(video, video_contains_first_frame)
        cond = self._check_cond(cond, video.shape[0])
        params = self._grad_params((video, cond), "encode", ff, video.shape[2], quantize)
        if params is not None:
            need_gvideo = video.is_floating_point() and video.requires_grad
            out, runner = self._grad_call("run_encode", video.contiguous(), cond, params, ff, quantize, need_gvideo)
            if not quantize:
                return out
            return (out, runner.codes) if self.use_fsq else (out, runner.codes, self.zero)
        with torch.no_grad():
            eng = self._tf32_engine()
            x = eng.encode_cl(video, ff, cond)
            if quantize:
                q, idx, _ = eng.quantize_cl(x)
                out = eng.to_channels_first(q)
                if self.use_fsq:
                    return out, idx
                return out, idx, self.zero
            return eng.to_channels_first(x)

    def _check_cond(self, cond, batch):
        """M:1542-1545 / M:1610-1613."""
        assert (not self.has_cond) or cond is not None, \
            "`cond` must be passed into tokenizer forward method since conditionable layers were specified"
        if cond is None:
            return None
        if not self.has_cond:
            return None                      # the reference runs the (Identity) stem and never uses the result
        assert tuple(cond.shape) == (batch, self.dim_cond)
        self._check_on_device(cond, "cond")
        return cond

    def _check_on_device(self, t, what):
        if t.device != self.device:
            raise RuntimeError(f"{what} is on {t.device} but the tokenizer is on {self.device}")

    def _decoded_frames(self, latent_frames, ff):
        """Frames of the reconstruction of `latent_frames` latent frames."""
        return latent_frames * self.time_downsample_factor - (self.time_padding if ff else 0)

    @_on_model_device
    @_precision_scope
    @_attn_dropout_scope
    def decode(self, quantized, cond=None, video_contains_first_frame=True):
        """M:1598-1649.  quantized: (B, C, T', H', W').  Differentiable (see _grad_params) wrt quantized, cond and the
        decoder's parameters (train.reached_parameters)."""
        assert quantized.ndim == 5 and quantized.shape[1] == self.quantizers.dim, \
            f"quantized must be (B, {self.quantizers.dim}, T, H, W), got {tuple(quantized.shape)}"
        self._check_on_device(quantized, "quantized")
        cond = self._check_cond(cond, quantized.shape[0])
        ff = bool(video_contains_first_frame)
        params = self._grad_params((quantized, cond), "decode", ff, self._decoded_frames(quantized.shape[2], ff))
        if params is not None:
            return self._grad_call("run_decode", quantized, cond, params, ff)[0]
        with torch.no_grad():
            eng = self._tf32_engine()
            return eng.decode_cl(eng.to_channels_last(quantized), ff, cond)

    @_on_model_device
    @_precision_scope
    @_attn_dropout_scope
    def decode_from_code_indices(self, codes, cond=None, video_contains_first_frame=True):
        """M:1579-1595.  Differentiable (see _grad_params) wrt cond and the parameters of decode and quantizers.project_out."""
        assert codes.dtype in (torch.long, torch.int32)                           # M:1585
        if codes.ndim == 2:                                                       # M:1587-1591
            n = codes.shape[-1]
            assert n % (self.fmap_size ** 2) == 0, \
                f"flattened video ids must have a length ({n}) that is divisible by the fmap size " \
                f"({self.fmap_size}) squared ({self.fmap_size ** 2})"
            codes = codes.reshape(codes.shape[0], -1, self.fmap_size, self.fmap_size)
        nc = self.quantizers.num_codebooks
        assert codes.ndim == (4 if nc == 1 else 5) and (nc == 1 or codes.shape[-1] == nc), \
            f"codes must be (B, T, H, W{'' if nc == 1 else ', num_codebooks'}) or flat (B, N), got {tuple(codes.shape)}"
        self._check_on_device(codes, "codes")
        ff = bool(video_contains_first_frame)
        cond = self._check_cond(cond, codes.shape[0])
        params = self._grad_params((cond,), "decode_codes", ff, self._decoded_frames(codes.shape[1], ff))
        if params is not None:
            return self._grad_call("run_decode_codes", codes.contiguous(), cond, params, ff)[0]
        with torch.no_grad():
            self._tf32_engine()
            return self._decode_codes_no_grad(codes, cond, ff)

    def _decode_codes_no_grad(self, codes, cond, ff):
        eng = self.engine
        if cond is not None:
            return self._graph_call("decode_codes_cond" + ("" if ff else "_noff"),
                                    lambda c, cd: eng.decode_cl(eng.codes_to_quantized_cl(c), ff, cd), codes.contiguous(), cond.contiguous())
        return self._graph_call("decode_codes" if ff else "decode_codes_noff",
                                lambda c: eng.decode_cl(eng.codes_to_quantized_cl(c), ff), codes.contiguous())

    @torch.no_grad()
    @_on_model_device
    @_precision_scope
    @_attn_dropout_scope
    def lfq_loss_breakdown(self, video, group=None):
        """Training-mode LFQ auxiliary terms the reference computes at M:1705 (``quantizer_loss_breakdown``):
        returns ``(codes, (per_sample_entropy, batch_entropy, commitment), aux_loss)``.  ``batch_entropy`` uses the
        cross-rank mean code probability -- the single all-reduce of the path (num_codebooks * codebook_size * 4 bytes) (dist.LfqBatchEntropy), issued
        on a side stream.  (The losses' backward and the GAN/perceptual terms are out of scope, SURVEY.md 8f N2.)"""
        from .dist import LfqBatchEntropy
        assert not self.use_fsq, "FSQ has no auxiliary loss (reference M:1702)"
        video, _ = self._check_video(video)
        eng = self._tf32_engine()
        x = eng.encode_cl(video)
        _, codes, pre = eng.quantize_cl(x, want_quantized=False, want_aux=True)
        q = self.quantizers
        be = LfqBatchEntropy(eng, num_codebooks=q.num_codebooks)
        be.start(pre, group)
        ps, bent, commit, aux = be.finish(q.diversity_gamma, q.entropy_loss_weight, q.commitment_loss_weight, group)
        return codes, (ps, bent, commit), aux

    def _forward_train_mode(self, eng, video, need_recon, ff=True, group=None):
        """``model.train()`` forward of the LFQ tokenizer (reference M:1705: ``self.quantizers(x, return_loss_breakdown=True)``
        in training mode): besides codes / reconstruction the quantiser's auxiliary terms are computed -- per-sample entropy,
        batch (codebook) entropy of the CROSS-RANK mean code probability, commitment -- and kept in
        ``self.quantizer_loss_breakdown`` = (per_sample_entropy, batch_entropy, commitment) / ``self.quantizer_aux_loss``.
        The batch-entropy term needs the one collective of the path: a SUM all-reduce of avg_prob (num_codebooks * codebook_size * 4 bytes) (A.1 step 7), issued
        on a side stream so that it overlaps the decoder.  The decoder is fed the quantised value q itself; the reference's
        straight-through ``x + (q - x).detach()`` equals q up to one rounding (SURVEY 8d cfg 3).  No autograd (N2)."""
        from .dist import LfqBatchEntropy
        qz = self.quantizers

        def enc(v):
            x = eng.encode_cl(v, ff)
            q, codes_, pre = eng.quantize_cl(x, want_quantized=need_recon, want_aux=True)
            return (codes_, pre, q) if need_recon else (codes_, pre)

        sfx = "" if ff else "_noff"
        res = self._graph_call(("train_enc_q" if need_recon else "train_enc") + sfx, enc, video)
        codes, pre = res[0], res[1]
        be = LfqBatchEntropy(eng, num_codebooks=qz.num_codebooks)
        be.start(pre, group)                                   # partial sums + all-reduce on the side stream ...
        recon = self._graph_call("train_dec" + sfx, lambda t: eng.decode_cl(t, ff), res[2]) if need_recon else None   # ... under the decoder
        ps, bent, commit, aux = be.finish(qz.diversity_gamma, qz.entropy_loss_weight, qz.commitment_loss_weight, group)
        self.quantizer_loss_breakdown = (ps, bent, commit)
        self.quantizer_aux_loss = aux
        return (codes, recon) if need_recon else codes

    def tokenize_stream(self, batch_size, cond=None, video_contains_first_frame=True):
        """A stream.TokenizeStream: push() chunks of a clip batch, get the codes one tokenize of the whole clip gives."""
        from .stream import TokenizeStream
        return TokenizeStream(self, batch_size, cond, video_contains_first_frame)

    def decode_stream(self, batch_size, cond=None, video_contains_first_frame=True):
        """A stream.DecodeStream: push() latent frames, get the frames one decode_from_code_indices of all of them gives."""
        from .stream import DecodeStream
        return DecodeStream(self, batch_size, cond, video_contains_first_frame)

    @torch.no_grad()
    def tokenize(self, video):
        """M:1651-1654."""
        self.eval()
        return self.forward(video, return_codes=True)

    @_on_model_device
    @_precision_scope
    @_attn_dropout_scope
    def forward(self, video_or_images, cond=None, return_loss=False, return_codes=False, return_recon=False,
                return_discr_loss=False, return_recon_loss_only=False, apply_gradient_penalty=True,
                video_contains_first_frame=True, adversarial_loss_weight=None,
                multiscale_adversarial_loss_weight=None):
        """The reference forward (M:1657-1896): inference returns (codes / reconstruction), ``return_recon_loss_only``,
        ``return_discr_loss`` and ``return_loss``: ``(total_loss, LossBreakdown)`` with ``total_loss = recon_loss + aux_loss *
        quantizer_aux_loss_weight + perceptual_loss * perceptual_loss_weight + gen_loss * adaptive_weight *
        adversarial_loss_weight + sum(multiscale_gen_losses * multiscale weights) * multiscale_adversarial_loss_weight``
        (M:1868-1896).  The perceptual term needs a ``vgg=`` module; the adaptive weights are the ratio of the perceptual and
        adversarial terms' gradient norms at ``conv_out.conv.weight`` in a train-mode step (M:1812-1868), 1 in eval mode.  The
        call-site ``adversarial_loss_weight`` / ``multiscale_adversarial_loss_weight`` default to the attributes; the
        discriminator step's total uses the attribute (M:1776-1779)."""
        assert (return_loss + return_codes + return_discr_loss) <= 1               # M:1674
        if return_discr_loss and self.discr is None:
            raise NotImplementedError("return_discr_loss needs the image discriminator, which is built for use_gan=True, "
                                      "adversarial_loss_weight > 0 and a `vgg=` module when the loss has a perceptual term "
                                      "(SURVEY.md 8f N2)")
        if return_loss and self._needs_gan_or_vgg():
            raise NotImplementedError(
                "return_loss with the perceptual term needs a `vgg=` module (this package downloads no VGG weights): pass "
                "vgg=<module> or construct with perceptual_loss_weight=0.")
        if return_loss and self.has_multiscale_discrs and not (self.has_gan or self.use_vgg):
            raise ValueError("the multiscale generator terms are taken on the image discriminator's or the perceptual term's "
                             "frame pick (M:1846-1850), and this model has neither (the reference fails with UnboundLocalError "
                             "here): construct with adversarial_loss_weight > 0 or pass a `vgg=` module")
        grad_step = (return_loss and self.training and torch.is_grad_enabled()
                     and any(p.requires_grad for p in self.parameters()))
        if self.dtype == torch.float16:
            # fp16 runs the no-grad tokenizer only: no gradients, and no discriminator or VGG (their paths train)
            if return_discr_loss:
                raise TypeError("return_discr_loss is not supported for float16 models: the discriminator has no fp16 path")
            if return_loss and (self.has_gan or self.use_vgg or self.has_multiscale_discrs):
                raise TypeError("return_loss is not supported for float16 models with a discriminator or a VGG: those modules "
                                "have no fp16 path")
            if grad_step:
                raise TypeError("a train-mode return_loss step with gradients is not supported for float16 models: run it under "
                                "torch.no_grad() or use float32 / bfloat16 parameters")
        if return_loss and self.training and self.use_vgg and (self.has_gan or self.has_multiscale_discrs) and not grad_step:
            raise RuntimeError("a train-mode return_loss with a VGG and a GAN needs gradients: the adaptive adversarial weight is "
                               "a ratio of gradient norms (M:1812-1841; the reference fails in torch.autograd.grad here)")
        video, ff = self._check_video(video_or_images, video_contains_first_frame)
        cond = self._check_cond(cond, video.shape[0])
        if adversarial_loss_weight is None:                                        # the call-site weights win (M:1671-1672)
            adversarial_loss_weight = self.adversarial_loss_weight
        if multiscale_adversarial_loss_weight is None:
            multiscale_adversarial_loss_weight = self.multiscale_adversarial_loss_weight
        if return_discr_loss:
            return self._discr_loss(video, ff, cond, apply_gradient_penalty)
        if grad_step:
            # the trainer's generator step (T:356-363): loss with a grad_fn.  Forward = the same kernels; backward = train.py
            from .train import TrainRunner, train_forward
            runner = TrainRunner(self)
            recon, aux, _, qlb = train_forward(self, video.contiguous(), ff, cond, runner=runner)
            target = video.float() / 255. if video.dtype == torch.uint8 else video
            recon_loss = torch.nn.functional.mse_loss(target.to(recon.dtype), recon)          # M:1722
            self.quantizer_loss_breakdown, self.quantizer_aux_loss = qlb, aux.detach()
            aux_losses = aux.to(recon_loss.dtype)
            total_loss = recon_loss + aux_losses * self.quantizer_aux_loss_weight                # M:1868-1871
            perceptual_loss, g_perc = self._perceptual_loss(target, recon)
            # the perceptual gradient norm at the last decoder layer, for the adaptive weights (M:1817-1820)
            norm_p = None
            if self.use_vgg and (self.has_gan or self.has_multiscale_discrs):
                norm_p = self._last_layer_grad_norm(runner, recon, *g_perc)
            gen_loss, g_gen = self._gen_loss(recon)
            adaptive_weight = 0.
            if self.has_gan:
                adaptive_weight = 1.
                if norm_p is not None:                                                             # M:1833-1841
                    w = self._adaptive_weight(norm_p, self._last_layer_grad_norm(runner, recon, *g_gen), 1e-3)
                    adaptive_weight = 1. if torch.isnan(w).any() else w
            ms_losses, ms_weights = self._multiscale_gen_terms(recon, g_gen if self.has_gan else g_perc, runner, norm_p)
            if self.use_vgg:
                total_loss = total_loss + perceptual_loss * self.perceptual_loss_weight
            if self.has_gan:
                total_loss = total_loss + gen_loss * adaptive_weight * adversarial_loss_weight   # M:1872-1875
            if self.has_multiscale_discrs:                                                         # M:1877-1881
                total_loss = total_loss + sum(l * w for l, w in zip(ms_losses, ms_weights)) * multiscale_adversarial_loss_weight
            return total_loss, LossBreakdown(recon_loss, aux_losses, qlb, perceptual_loss, gen_loss, adaptive_weight,
                                             ms_losses, ms_weights)
        with torch.no_grad():
            # a loss with a discriminator or a VGG term stays IEEE: those modules train, and their inputs with them
            eng = self._tf32_engine(follow=not (return_loss and (self.has_gan or self.use_vgg or self.has_multiscale_discrs)))
            need_recon = return_recon or return_recon_loss_only or return_loss or not return_codes
            out, aux = self._no_grad_forward(eng, video, ff, cond, need_recon)
            if return_codes and not return_recon:
                return out                                                         # M:1707-1708
            codes, recon = out
            if return_codes:
                return codes, recon                                                # M:1714-1715
            if not (return_loss or return_recon_loss_only):
                return recon                                                       # M:1719-1720
            recon_loss = eng.mse(video, recon).to(self.dtype)                      # M:1722
            if return_recon_loss_only:                                             # M:1726-1727
                return recon_loss, recon
            # M:1868-1896: perceptual_loss = zero without a VGG; gen_loss = zero and adaptive_weight = 0. without a
            # discriminator, adaptive_weight = 1. with one, and every multiscale weight 1. (no gradients here, M:1833, M:1861)
            zero = self.zero
            aux_losses = zero if aux is None else aux.to(recon_loss.dtype)         # eval mode / FSQ: M:1700-1703
            total_loss = recon_loss + aux_losses * self.quantizer_aux_loss_weight
            perceptual_loss, g_perc = self._perceptual_loss(video.float() / 255. if video.dtype == torch.uint8 else video, recon)
            if self.use_vgg:
                total_loss = total_loss + perceptual_loss * self.perceptual_loss_weight
            gen_loss, g_gen = self._gen_loss(recon)
            adaptive_weight = 1. if self.has_gan else 0.
            if self.has_gan:
                total_loss = total_loss + gen_loss * adaptive_weight * adversarial_loss_weight
            ms_losses, ms_weights = self._multiscale_gen_terms(recon, g_gen if self.has_gan else g_perc)
            if self.has_multiscale_discrs:
                total_loss = total_loss + sum(l * w for l, w in zip(ms_losses, ms_weights)) * multiscale_adversarial_loss_weight
            qlb = None if (self.use_fsq or aux is None) else self.quantizer_loss_breakdown
            return total_loss, LossBreakdown(recon_loss, aux_losses, qlb, perceptual_loss, gen_loss, adaptive_weight,
                                             ms_losses, ms_weights)

    def _no_grad_forward(self, eng, video, ff, cond, need_recon):
        """The tokenizer forward without gradients -> (codes | (codes, recon), train-mode LFQ aux loss | None)."""
        aux = None

        def run(v, cd=None):
            x = eng.encode_cl(v, ff, cd)
            q, codes_, _ = eng.quantize_cl(x, want_quantized=need_recon)
            if not need_recon:
                return codes_
            return codes_, eng.decode_cl(q, ff, cd)

        if cond is not None:
            out = self._graph_call(("fwd_recon_cond" if need_recon else "fwd_codes_cond") + ("" if ff else "_noff"), run,
                                   video.contiguous(), cond.contiguous())
        elif self.training and not self.use_fsq:
            out = self._forward_train_mode(eng, video.contiguous(), need_recon, ff)
            aux = self.quantizer_aux_loss
        else:
            out = self._graph_call(("fwd_recon" if need_recon else "fwd_codes") + ("" if ff else "_noff"), run, video.contiguous())
        return out, aux

    @staticmethod
    def _pick_frames(video, frame_indices):
        """pick_video_frame (M:91-98): (B, C, F, H, W), indices (B, 1) -> (B, C, H, W)."""
        b = torch.arange(video.shape[0], device=video.device)[:, None]
        return video.transpose(1, 2)[b, frame_indices.to(video.device)][:, 0]

    def _gen_loss(self, recon):
        """The adversarial generator term (M:1826-1831): -discr(frames).mean() on one random frame per clip, drawn from the
        default CPU generator as the reference does -> (loss, (frame indices, d loss / d frames | None)); (zero, None)
        without a discriminator."""
        if not self.has_gan:
            return self.zero, None
        from .gan import generator_term
        frame_indices = torch.randn((recon.shape[0], recon.shape[2])).topk(1, dim=-1).indices
        loss, info = generator_term(self.discr, self._pick_frames(recon, frame_indices))
        return loss, (frame_indices, info.get("grad_images"))

    def _perceptual_loss(self, target, recon):
        """The perceptual term (M:1788-1808): F.mse_loss of the VGG features of one random frame per clip (drawn before the
        generator term's, M:1792) of the target and the reconstruction -> (loss, (frame indices, d loss / d recon frames |
        None)); (zero, None) without a VGG."""
        if not self.use_vgg:
            return self.zero, None
        from .vgg import perceptual_loss
        frame_indices = torch.randn((recon.shape[0], recon.shape[2])).topk(1, dim=-1).indices
        real = self._pick_frames(target, frame_indices).to(self.dtype).contiguous()
        loss, info = perceptual_loss(self.vgg, real, self._pick_frames(recon, frame_indices), self.channels, self._vgg_cache)
        return loss, (frame_indices, info.get("grad_frames"))

    @staticmethod
    def _scatter_frames(recon, frame_indices, g_frames):
        """The reconstruction gradient of a loss on the picked frames (B, C, H, W): zero on every other frame."""
        g = torch.zeros(recon.shape, device=recon.device, dtype=g_frames.dtype)
        g.transpose(1, 2)[torch.arange(recon.shape[0], device=recon.device), frame_indices[:, 0].to(recon.device)] = g_frames
        return g

    def _last_layer_grad_norm(self, runner, recon, frame_indices, g_frames):
        """|d loss / d W|, W = conv_out.conv.weight, for a loss on the picked reconstruction frames with gradient g_frames,
        from the tokenizer's saved activations (TrainRunner.last_layer_weight_grad) -- no backward runs."""
        return runner.last_layer_weight_grad(self._scatter_frames(recon, frame_indices, g_frames)).norm(p=2)

    @staticmethod
    def _adaptive_weight(norm_p, norm_g, eps):
        """M:1836-1838 / M:1864-1866: norm_p / max(norm_g, eps), clamped at 1e3."""
        return (norm_p / norm_g.clamp(min=eps)).clamp(max=1e3).detach()

    def _multiscale_gen_terms(self, recon, picked, runner=None, norm_p=None):
        """The multiscale generator terms (M:1846-1866) -> (losses, adaptive weights), one of each per multiscale
        discriminator; ([], []) without them.  The reference's loop sets ``fake_logits = recon_video_frames`` and never calls
        the discriminator, so every loss is hinge_gen_loss(frames) = -frames.mean() of the same picked reconstruction frames
        (picked: the image-GAN term's (frame indices, ...), or the perceptual term's without an image GAN) -- no new random
        draw.  Every weight is then the same: norm_p over the loss's last-layer gradient norm (clamped at 1e-5, no NaN
        fallback) when the perceptual norm norm_p exists, else 1."""
        if not self.has_multiscale_discrs:
            return [], []
        frame_indices = picked[0]
        frames = self._pick_frames(recon, frame_indices)
        loss = -frames.mean()
        weight = 1.
        if norm_p is not None:
            g_frames = torch.full(frames.shape, -1. / frames.numel(), device=recon.device, dtype=recon.dtype)
            weight = self._adaptive_weight(norm_p, self._last_layer_grad_norm(runner, recon, frame_indices, g_frames), 1e-5)
        n = len(self.multiscale_discrs)
        return [loss] * n, [weight] * n

    def _discr_loss(self, video, ff, cond, apply_gradient_penalty):
        """``return_discr_loss`` (M:1731-1786): the tokenizer runs without gradients (as the no-grad forward, including the
        train-mode LFQ all-reduce), then the hinge loss of the device discriminator on one real and one reconstructed frame
        per clip, the hinge loss of each multiscale discriminator on the whole real and reconstructed videos (torch runs the
        user's modules; a uint8 video is passed as x / 255 in the model's dtype), plus the image discriminator's gradient
        penalty (gan.gradient_penalty) when asked for."""
        from .gan import DiscrLossBreakdown, gradient_penalty
        with torch.no_grad():
            (_, recon), _ = self._no_grad_forward(self.engine, video, ff, cond, True)
        frame_indices = torch.randn((video.shape[0], video.shape[2])).topk(1, dim=-1).indices
        frames = video.float() / 255. if video.dtype == torch.uint8 else video
        real = self._pick_frames(frames, frame_indices).to(self.dtype).contiguous()
        fake = self._pick_frames(recon, frame_indices).detach().contiguous()
        real_logits, fake_logits = self.discr(real), self.discr(fake)
        discr_loss = _hinge_discr_loss(fake_logits, real_logits)
        multiscale = [self.zero]
        if self.has_multiscale_discrs:                                                     # M:1752-1765
            real_video = frames.to(self.dtype) if video.dtype == torch.uint8 else video
            fake_video = recon.detach()
            multiscale = []
            for d in self.multiscale_discrs:
                real_ms = d(real_video)
                multiscale.append(_hinge_discr_loss(d(fake_video), real_ms))
        if apply_gradient_penalty:
            gp = gradient_penalty(self.discr, real) + gradient_penalty(self.discr, fake)
        else:
            gp = self.zero
        total = discr_loss + gp * self.grad_penalty_loss_weight + sum(multiscale) * self.multiscale_adversarial_loss_weight
        return total, DiscrLossBreakdown(discr_loss, multiscale, gp)

    def _has_vgg(self) -> bool:
        """True when the reference constructor would have built a VGG (M:1392)."""
        return bool(self.channels in {1, 3, 4} and self.perceptual_loss_weight > 0.)

    def _needs_gan_or_vgg(self) -> bool:
        """True when the loss needs a term this package does not build: the perceptual term without a VGG module (M:1392),
        or the GAN term of a model that built no discriminator (M:1427)."""
        return bool((self._has_vgg() and not self.use_vgg) or (self.use_gan and self.adversarial_loss_weight > 0. and self.discr is None))

    @property
    def dtype(self):
        return self.conv_in.conv.weight.dtype
