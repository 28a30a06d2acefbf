"""Host-side executor: walks the VideoTokenizer layer schedule and launches the sm_90a
kernels of libmagvit2_b200.so through the C ABI (ctypes).  PyTorch is used only for device
memory (caching allocator), streams and parameter storage.

Activations are channels-last (B, T, H, W, C) tensors in the compute dtype (fp32 -> CUDA-core
path, or TF32 wgmma while torch allows TF32 matmuls; bf16 or fp16 -> wgmma tensor-core path for the dense contractions,
tensor_core_dtype).  There is no eager / CPU
fallback: every op is a library call and a missing library is an error.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch

from . import _lib
from ._lib import (ACT_ELU, ACT_NONE, ACT_SILU, MV2_BF16, MV2_F16, MV2_F32, MV2_TF32, MV2_U8, SHUFFLE_NONE, SHUFFLE_SPACE,
                   SHUFFLE_TIME, AttnArgs, ConvArgs, ConvHist, TcConvArgs, TcRuArgs, check)


def _dt(t: torch.dtype) -> int:
    if t == torch.float32:
        return MV2_F32
    if t == torch.bfloat16:
        return MV2_BF16
    if t == torch.float16:
        return MV2_F16
    raise TypeError(f"unsupported dtype {t} (only float32, bfloat16 and float16)")


def tensor_core_dtype(t: torch.dtype, tf32: bool = False) -> bool:
    """True for the parameter dtypes whose dense contractions run on the wgmma tensor cores: bf16 and fp16 (16-bit
    storage, fp32 accumulation) always, fp32 with `tf32` (fp32 storage, TF32 multiply, fp32 accumulation); otherwise fp32
    runs on the CUDA cores."""
    return t in (torch.bfloat16, torch.float16) or (tf32 and t == torch.float32)


def tf32_matmul_enabled() -> bool:
    """torch's TF32 switch for fp32 matmuls (torch.set_float32_matmul_precision("high" / "medium"),
    torch.backends.cuda.matmul.allow_tf32 = True or fp32_precision = "tf32"), which an fp32 tokenizer's calls without
    gradients follow.  cuDNN's conv switch, on by default, is not followed: it would change every fp32 result."""
    return torch.backends.cuda.matmul.fp32_precision == "tf32"


def _src_dt(t: torch.dtype) -> int:
    """dtype code of a layout-in SOURCE tensor: uint8 frames are accepted there (normalised x / 255 on the fly)."""
    return MV2_U8 if t == torch.uint8 else _dt(t)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


class AttnDropout:
    """Attention dropout of one train-mode tokenizer forward: drop probability p, the 64-bit Philox seed of the forward and
    the index of the next softmax attention call (its `call`, in execution order: encoder stages, then decoder stages).
    (seed, call) selects the call's keep mask (include/magvit2_b200.h, mv2_dropout_args)."""

    def __init__(self, p: float, seed: int):
        self.p, self.seed, self.calls = float(p), int(seed), 0

    def take(self) -> _lib.DropoutArgs:
        """The dropout arguments of the next attention call."""
        a = _lib.DropoutArgs(seed=self.seed, call=self.calls, p=self.p)
        self.calls += 1
        return a


class StreamState:
    """Causal state of a streamed clip batch (stream.py), carried from one push to the next: per layer, the history frames
    of a causal conv, the previous frame of a token shift, the time attention's K/V cache and output buffers, the gateloop
    scan state.  A view with a key prefix (`sub`) is what the layer functions receive; None everywhere means a whole-clip
    call.  Every buffer a push's kernels read or write across pushes is allocated once and updated in place, so a push
    captured as a CUDA graph (stream.PushPlan) can be replayed on later pushes; only the K/V cache moves when it grows, and
    the host steps that use it are not captured."""

    def __init__(self, slots=None, prefix=""):
        self._slots = {} if slots is None else slots
        self._prefix = prefix

    def sub(self, name) -> "StreamState":
        return StreamState(self._slots, f"{self._prefix}{name}/")

    def get(self, name):
        return self._slots.get(self._prefix + name)

    def put(self, name, value):
        self._slots[self._prefix + name] = value

    def history_counts(self):
        """The frame count of every conv history, in layer order: with the chunk's shape, what a push's launches depend on
        besides the time attention's K/V cache length."""
        return tuple(v[1] for k, v in self._slots.items() if k.rsplit("/", 1)[-1] == "hist")

    def kv_capacities(self):
        """The frame capacity of every time attention's K/V cache, in layer order."""
        return tuple(v[0].shape[1] for k, v in self._slots.items() if k.rsplit("/", 1)[-1] == "kv")

    def restart_rows(self, rows):
        """Starts clip rows `rows` over: the next push computes for them what the first push of a new stream computes.
        Their slices of every conv history, token-shift frame and gateloop scan state are zeroed in place (zero history
        frames give the values of the causal padding, DESIGN.md 3.7), and each time attention's K/V cache records the
        current end of the cache as where their keys start.  No buffer moves and no frame count changes, so a push
        captured as a CUDA graph replays unchanged."""
        rows = set(rows)
        for k, v in self._slots.items():
            leaf = k.rsplit("/", 1)[-1]
            if leaf in ("hist", "prev", "s"):
                buf = v[0] if leaf == "hist" else v
                for r0, r1, hit in row_runs([r in rows for r in range(buf.shape[0])]):
                    if hit:
                        buf[r0:r1].zero_()
            elif leaf == "kv":
                buf, L, starts = v
                self._slots[k] = (buf, L, tuple(L if r in rows else s for r, s in enumerate(starts)))


def row_runs(starts):
    """[(first row, end row, value)] of the runs of consecutive rows with equal `starts` values, in row order."""
    runs = []
    for r, s in enumerate(starts):
        if runs and runs[-1][2] == s:
            runs[-1] = (runs[-1][0], r + 1, s)
        else:
            runs.append((r, r + 1, s))
    return runs


def kv_cache_plan(length, T, starts, step):
    """When a K/V cache holding `length` frames has no room for T more: (frames to drop from its front, new capacity).
    The frames before the earliest row start belong to no live clip; the capacity is the rest plus T, rounded up to a
    multiple of `step`."""
    drop = min(starts)
    return drop, _round_up(length - drop + T, step)


def _sub(ss: Optional[StreamState], name):
    return None if ss is None else ss.sub(name)


@dataclass
class ConvPack:
    """One convolution's parameters in kernel layout."""
    w: torch.Tensor              # [taps][Ci][Co] in the compute dtype (CUDA-core path)
    bias: Optional[torch.Tensor]  # fp32 [Co]
    k: Tuple[int, int, int]
    Ci: int
    Co: int
    w_tc: Optional[torch.Tensor] = None      # [Co][taps*Ci] bf16 / fp16 / fp32 (TF32), K-major (wgmma path); rows permuted for shuffles
    bias_tc: Optional[torch.Tensor] = None   # bias in w_tc's row order
    Ci_tc: int = 0                           # GEMM dims of the wgmma call (may be padded / re-paired)
    Co_tc: int = 0
    epi_mode: int = 0                        # 1: fused GEGLU (output has Co_tc // 2 channels); 2: (act(conv) + res) * 2^-0.5
    k_tc: Optional[Tuple[int, int, int]] = None
    macs: int = 0                            # algorithmic multiply-accumulates per output position (Co * Ci * taps, unpadded)
    w_down: Optional[torch.Tensor] = None    # SpatialDownsample2x pack for mv2_tc_down_space_forward ([Co][6][2*Ci], as w_tc)


def pack_conv(weight: torch.Tensor, bias: Optional[torch.Tensor], dtype, k=None, shuffle_q: int = 1, tc=None) -> ConvPack:
    """weight: torch layout (Co, Ci, *kernel).  Kernel dims are mapped onto (kt, kh, kw) by `k`.
    shuffle_q = 4 / 2 for the depth-to-space / depth-to-time up-samplers: the wgmma kernel wants output
    rows ordered (q, c) instead of the reference's (c, q) so shuffled stores are channel-contiguous.
    tc: build the wgmma pack too (default: tensor_core_dtype(dtype); True for an fp32 model's TF32 pack)."""
    if tc is None:
        tc = tensor_core_dtype(dtype)
    Co, Ci = weight.shape[:2]
    if k is None:
        ks = tuple(weight.shape[2:])
        k = (1,) * (3 - len(ks)) + ks
    w3 = weight.detach().reshape(Co, Ci, -1)
    w = w3.permute(2, 1, 0).contiguous().to(dtype)
    b = None if bias is None else bias.detach().float().contiguous()
    pk = ConvPack(w=w, bias=b, k=tuple(int(v) for v in k), Ci=int(Ci), Co=int(Co))
    pk.macs = int(Co) * int(Ci) * int(w3.shape[2])
    if tc:
        wt = w3.permute(0, 2, 1).reshape(Co, -1)                      # [Co][tap*Ci + ci]
        bt = b
        if shuffle_q > 1:
            cy = Co // shuffle_q
            wt = wt.reshape(cy, shuffle_q, -1).permute(1, 0, 2).reshape(Co, -1)
            bt = None if b is None else b.reshape(cy, shuffle_q).t().reshape(Co).contiguous()
        pk.w_tc = wt.contiguous().to(dtype)
        pk.bias_tc = bt
        pk.Ci_tc, pk.Co_tc, pk.k_tc = pk.Ci, pk.Co, pk.k
    return pk


def pack_conv_down_space(pk: ConvPack, weight):
    """SpatialDownsample2x (M:768: Conv2d k3 s2 p1) for mv2_tc_down_space_forward: w[co][tap'][2*Ci], tap' = dh * 2 + q,
    q = 0 -> [zeros | w[:, :, dh, 0]] (the column left of the pair), q = 1 -> [w[:, :, dh, 1] | w[:, :, dh, 2]]."""
    Co, Ci, kh, kw = weight.shape
    if (kh, kw) != (3, 3) or Ci * pk.w_tc.element_size() % 128 != 0 or Co % 32 != 0:     # 128-byte K rows
        return
    w = weight.detach().float()
    wd = torch.zeros((Co, 3, 2, 2 * Ci), device=w.device)
    wd[:, :, 0, Ci:] = w[:, :, :, 0].permute(0, 2, 1)
    wd[:, :, 1, :Ci] = w[:, :, :, 1].permute(0, 2, 1)
    wd[:, :, 1, Ci:] = w[:, :, :, 2].permute(0, 2, 1)
    pk.w_down = wd.reshape(Co, 6 * 2 * Ci).contiguous().to(pk.w_tc.dtype)


def _adopt_tc_packs(old, new):
    """Sets the wgmma fields of every ConvPack in the pack tree `old` to those of its counterpart in `new`, a tree of the
    same parameters packed with them; old's CUDA-core tensors stay as they are."""
    if isinstance(old, ConvPack):
        for f in ("w_tc", "bias_tc", "Ci_tc", "Co_tc", "epi_mode", "k_tc", "w_down"):
            setattr(old, f, getattr(new, f))
    elif isinstance(old, dict):
        for k, v in new.items():
            if old.get(k) is None:          # a wgmma-only pack (the kw-packed conv_in)
                old[k] = v
            else:
                _adopt_tc_packs(old[k], v)


def _round_up(v, m):
    return (v + m - 1) // m * m


def pack_ff(fc1_w, fc1_b, fc2_w, fc2_b, dtype, tc=None):
    """FeedForward weights (reference M:492-496).  wgmma layout: the hidden width I is padded to a multiple of 64,
    fc1's rows are re-paired as [8 x-rows, their 8 gate-rows] per group of 16 so GEGLU (M:466-469) fuses into fc1's
    epilogue, and fc2's K is zero-padded to match.  The fused fc1 needs K = C a multiple of 16; for other widths there
    are no wgmma packs, and fc1, GEGLU and fc2 run unfused on the CUDA cores."""
    tc = tensor_core_dtype(dtype) if tc is None else tc
    fc1 = pack_conv(fc1_w, fc1_b, dtype, tc=tc)
    fc2 = pack_conv(fc2_w, fc2_b, dtype, tc=tc)
    two_i, C_ = fc1_w.shape[:2]
    if tc and C_ % 16 != 0:
        for pk in (fc1, fc2):
            pk.w_tc = pk.bias_tc = None
    elif tc:
        I = two_i // 2
        Ip = _round_up(I, 64)
        w1 = fc1_w.detach().reshape(two_i, C_).float()
        b1 = fc1_b.detach().float()
        wx = torch.zeros((Ip, C_), device=w1.device)
        wg = torch.zeros((Ip, C_), device=w1.device)
        bx = torch.zeros((Ip,), device=w1.device)
        bg = torch.zeros((Ip,), device=w1.device)
        wx[:I], wg[:I], bx[:I], bg[:I] = w1[:I], w1[I:], b1[:I], b1[I:]
        wp = torch.stack((wx.reshape(Ip // 8, 8, C_), wg.reshape(Ip // 8, 8, C_)), dim=1).reshape(2 * Ip, C_)
        bp = torch.stack((bx.reshape(Ip // 8, 8), bg.reshape(Ip // 8, 8)), dim=1).reshape(2 * Ip)
        fc1.w_tc, fc1.bias_tc = wp.contiguous().to(dtype), bp.contiguous()
        fc1.Ci_tc, fc1.Co_tc, fc1.epi_mode = int(C_), 2 * Ip, 1
        w2 = fc2_w.detach().reshape(fc2_w.shape[0], I).float()
        w2p = torch.zeros((w2.shape[0], Ip), device=w2.device)
        w2p[:, :I] = w2
        fc2.w_tc = w2p.contiguous().to(dtype)
        fc2.Ci_tc, fc2.Co_tc = Ip, int(w2.shape[0])
    return fc1, fc2


def pack_linear_attention(la, dt, tc=None):
    """LinearSpaceAttention (M:390-442) for Engine.linear_attention."""
    return dict(gamma=la.norm.gamma.detach().float().contiguous(),
                q=pack_conv(la.attn.to_q[0].weight[:, :, None, None, None], None, dt, tc=tc),
                kv=pack_conv(la.attn.to_kv[0].weight[:, :, None, None, None], None, dt, tc=tc),
                out=pack_conv(la.attn.to_out[0].weight[:, :, None, None, None], None, dt, tc=tc),
                heads=la.heads, dim_head=la.dim_head)


def pack_feed_forward(ff, dt, tc=None):
    """FeedForward (M:471-496) for Engine.feed_forward."""
    fc1, fc2 = pack_ff(ff.net[0].weight, ff.net[0].bias, ff.net[2].weight, ff.net[2].bias, dt, tc=tc)
    return dict(gamma=ff.norm.gamma.detach().float().reshape(-1).contiguous(), fc1=fc1, fc2=fc2, inner=ff.dim_inner)


def pack_conv_in_kwpack(weight, bias, cpack=32, dtype=torch.bfloat16):
    """conv_in (M:1109) for the wgmma path: (Co, Cin, kt, kh, kw) -> [Co][(dt, dh)][dw * Cin + c], zero padded to
    `cpack` channels -- pairs with mv2_ingest_kwpack."""
    Co, Cin, kt, kh, kw = weight.shape
    if Cin * kw > cpack:
        return None
    w = weight.detach().float().permute(0, 2, 3, 4, 1).reshape(Co, kt * kh, kw * Cin)
    wp = torch.zeros((Co, kt * kh, cpack), device=w.device)
    wp[:, :, :kw * Cin] = w
    pk = ConvPack(w=None, bias=None, k=(kt, kh, 1), Ci=cpack, Co=int(Co))
    pk.w_tc = wp.reshape(Co, kt * kh * cpack).contiguous().to(dtype)
    pk.bias_tc = None if bias is None else bias.detach().float().contiguous()
    pk.Ci_tc, pk.Co_tc, pk.k_tc = cpack, int(Co), (kt, kh, 1)
    pk.kw_orig, pk.cin_orig = int(kw), int(Cin)
    pk.macs = int(Co) * int(Cin) * int(kt * kh * kw)          # the padded K (cpack x kt x kh) is not algorithmic work
    return pk


def param_signature(module):
    """Identity of a module's parameter storage: changes on load_state_dict, .to(), optimizer steps and in-place edits."""
    ps = list(module.parameters())
    return (tuple((p.data_ptr(), p._version) for p in ps), ps[0].dtype, ps[0].device)


class PackCache:
    """The engine and weight packs of a module that runs on an engine of its own (the discriminator, the VGG,
    CausalConvTranspose3d).  The engine outlives re-packs, so its `launches` keep counting; copies and pickles start empty,
    as its ctypes handles belong to this instance."""

    def __init__(self):
        self.engine: Optional[Engine] = None
        self.packs = None
        self._sig = None

    def get(self, module, what, build, key=(), half=False):
        """-> (engine, packs): re-packs with build(engine), under no_grad, when the module's parameters (param_signature) or
        `key` changed, after binding the engine to them (Engine.bind; `what` names the module in its errors, `half` admits
        fp16 parameters)."""
        sig = (param_signature(module), key)
        if sig != self._sig:
            self._sig = None
            if self.engine is None:
                self.engine = Engine(None)
            self.engine.bind(next(iter(module.parameters())), what, half)
            with torch.no_grad():
                self.packs = build(self.engine)
            self._sig = sig
        return self.engine, self.packs

    def __reduce__(self):         # pickle, copy and deepcopy
        return PackCache, ()


class Engine:
    """Executes the inference path of one VideoTokenizer on its parameters' device/dtype."""

    def __init__(self, model):
        self.model = model
        self.lib = _lib.load()
        self._packs: Dict[str, object] = {}
        self._sig = None
        self._sig_id = 0             # bumped whenever parameters are re-packed (invalidates cached CUDA graphs)
        self.launches = 0            # kernels launched through the C ABI (bench's gpu_launches)
        self.use_tc = True           # bf16 / fp16: dense contractions on wgmma (False -> CUDA-core cross-check path)
        # fp32: the current call runs its dense contractions on the TF32 wgmma kernels (set per call by the model, from
        # torch's switch, for calls without gradients only; the packs they read are added by prepare(tf32_packs=True))
        self.tf32 = False
        self._tf32_packs = False
        self.tc_variant = "auto"     # "auto" (Engine.conv_kernel's choice) | "tap" (tc_conv.cu only)
        self.fuse_ru = True          # bf16 / fp16: conv3x3x3 + ELU + conv1x1x1 + ELU + SE pool partials in one wgmma launch (C = 64 / 128)
        self.fused_ru_calls = 0
        self.tc_calls = 0
        self.slab_calls = 0
        self.simt_conv_calls = 0
        self.taps: Optional[dict] = None  # when set, per-stage activations are recorded (tests)
        self._prof: Optional[list] = None  # when set, (event0, event1, flops) per wgmma conv launch
        self.conv_log: Optional[list] = None  # when set, one record per tensor-core conv launch (Engine._conv_launch)
        self.dropout: Optional[AttnDropout] = None  # set for the duration of a train-mode forward with attention dropout
        # set while a stream push is captured (stream.PushPlan): host_step(step) runs step(), a piece of the push that a
        # CUDA graph cannot replay, between two captured segments and returns its result
        self.host_step: Optional[Callable] = None

    # ------------------------------------------------------------------ parameters
    def bind(self, p0: torch.Tensor, what: str, half: bool = True):
        """Runs on the device and in the dtype of parameter p0, after checking that they are an sm_90 CUDA device and
        fp32 / bf16 / fp16 (fp16 only with `half`: the modules that only train, the discriminator and the VGG, have no
        fp16 path).  `what` names the model in the error messages."""
        if p0.device.type != "cuda":
            raise RuntimeError(f"{what} runs on CUDA (sm_90a) only; move the model with .cuda() -- there is no CPU fallback")
        if p0.dtype == torch.float16 and not half:
            raise TypeError(f"{what} does not run in float16 (its training path has no fp16 support): use float32 or bfloat16")
        if p0.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise TypeError("parameters must be float32, bfloat16 or float16")
        arch = self.lib.mv2_device_arch()
        if arch != 90:
            raise RuntimeError(f"libmagvit2_b200.so targets sm_90a (H100); device reports sm_{arch}")
        self.dtype = p0.dtype
        self.device = p0.device

    def prepare(self, tf32_packs: bool = False):
        """(Re)pack parameters into kernel layouts when they changed (load_state_dict, .to(), ...).  An fp32 model's TF32
        packs are built on the first call that needs them (tf32_packs, or self.tf32) and kept next to its CUDA-core packs
        until the next re-pack; adding them leaves every existing pack tensor, and with it every captured graph, valid."""
        sig = param_signature(self.model)
        tf32_packs = (tf32_packs or self.tf32) and sig[1] == torch.float32
        if sig == self._sig:
            if tf32_packs and not self._tf32_packs:
                _adopt_tc_packs(self._packs, self._build_packs(True))
                self._tf32_packs = True
            return
        self.bind(self.model.conv_in.conv.weight, "magvit2_pytorch_b200.VideoTokenizer")
        self._packs = self._build_packs(tensor_core_dtype(self.dtype, tf32_packs))
        self._tf32_packs = tf32_packs
        self._sig = sig
        self._sig_id += 1

    def _build_packs(self, tc: bool) -> Dict[str, object]:
        """Every parameter of the model in kernel layout; tc: with the wgmma packs (bf16 / fp16, or an fp32 model's TF32)."""
        m = self.model
        dt = self.dtype
        P: Dict[str, object] = {}
        P["conv_in"] = pack_conv(m.conv_in.conv.weight, m.conv_in.conv.bias, dt, tc=tc)
        P["conv_in_tc"] = pack_conv_in_kwpack(m.conv_in.conv.weight, m.conv_in.conv.bias, dtype=dt) if tc else None
        P["conv_out"] = pack_conv(m.conv_out.conv.weight, m.conv_out.conv.bias, dt, tc=tc)
        if m.separate_first_frame_encoding:       # SameConv2d (M:887-890): a (1, kh, kw) conv on the single first frame
            P["conv_in_ff"] = pack_conv(m.conv_in_first_frame.weight, m.conv_in_first_frame.bias, dt, tc=tc)
            P["conv_out_ff"] = pack_conv(m.conv_out_first_frame.weight, m.conv_out_first_frame.bias, dt, tc=tc)

        def f32(t):
            return t.detach().float().contiguous()

        def pack_ru(ru, key):
            seq = ru.fn
            se = seq[4]
            C_ = seq[2].weight.shape[0]
            P[key] = dict(
                conv3=pack_conv(seq[0].conv.weight, seq[0].conv.bias, dt, tc=tc),
                conv1=pack_conv(seq[2].weight, seq[2].bias, dt, tc=tc),
                wk=f32(se.to_k.weight.reshape(-1)), bk=float(se.to_k.bias.detach().float().item()),
                w1=f32(se.net[0].weight.reshape(se.net[0].weight.shape[0], C_)), b1=f32(se.net[0].bias),
                w2=f32(se.net[2].weight.reshape(C_, -1)), b2=f32(se.net[2].bias),
                hidden=int(se.net[0].weight.shape[0]),
            )

        def pack_ffn(ff, key):
            P[key] = pack_feed_forward(ff, dt, tc)

        def pack_attn(at, key):
            P[key] = dict(gamma=f32(at.norm.gamma), qkv=pack_conv(at.to_qkv[0].weight[:, :, None, None, None], None, dt, tc=tc),
                          out=pack_conv(at.to_out[1].weight[:, :, None, None, None], None, dt, tc=tc),
                          mem_kv=at.mem_kv.detach().to(dt).float().contiguous(),
                          heads=at.heads, dim_head=at.dim_head, n_mem=int(at.mem_kv.shape[2]))

        def pack_lin(la, key):
            P[key] = pack_linear_attention(la, dt, tc)

        for side, layers in (("enc", m.encoder_layers), ("dec", m.decoder_layers)):
            stages = m.stages if side == "enc" else list(reversed(m.stages))
            for i, st in enumerate(stages):
                mod = layers[i]
                key = f"{side}{i}"
                if st.kind == "residual":
                    units = list(mod) if st.nested else [mod]
                    for j, ru in enumerate(units):
                        pack_ru(ru, f"{key}.{j}")
                elif st.kind == "cond_residual":
                    w = mod.conv.weights
                    wq = w.detach().to(dt).float()                  # the weights as the module holds them in this dtype
                    P[key] = dict(conv3=pack_conv(w, None, dt, tc=tc), conv1=pack_conv(mod.conv_out.weight, mod.conv_out.bias, dt, tc=tc),
                                  S=(wq * wq).sum(dim=(2, 3, 4)).contiguous(), eps=float(mod.conv.eps),
                                  wc=f32(mod.to_cond.weight), bc=f32(mod.to_cond.bias))
                elif st.kind == "compress_space":
                    if side == "enc":
                        P[key] = pack_conv(mod.conv.weight, mod.conv.bias, dt, tc=tc)                     # (Co,Ci,3,3) -> k=(1,3,3)
                        if tc:
                            pack_conv_down_space(P[key], mod.conv.weight)
                    else:
                        P[key] = pack_conv(mod.net[0].weight, mod.net[0].bias, dt, shuffle_q=4, tc=tc)    # (4Co,Ci,1,1)
                elif st.kind == "compress_time":
                    if side == "enc":
                        P[key] = pack_conv(mod.conv.weight, mod.conv.bias, dt, k=(3, 1, 1), tc=tc)        # Conv1d (Co,Ci,3)
                    else:
                        P[key] = pack_conv(mod.net[0].weight, mod.net[0].bias, dt, k=(1, 1, 1), shuffle_q=2, tc=tc)  # Conv1d (2Co,Ci,1)
                elif st.kind == "attend_space":
                    pack_attn(mod[0].fn, key + ".attn")
                    pack_ffn(mod[1].fn, key + ".ff")
                elif st.kind == "attend_time":
                    pack_attn(mod[0].fn.fn, key + ".attn")
                    pack_ffn(mod[1].fn.fn, key + ".ff")
                elif st.kind == "linear_attend_space":
                    pack_lin(mod[0].fn, key + ".attn")
                    pack_ffn(mod[1].fn, key + ".ff")
                elif st.kind == "gateloop_time":
                    gl = mod.fn.fn
                    P[key] = dict(gamma=f32(gl.norm.gamma), qkva=pack_conv(gl.to_qkva[0].weight[:, :, None, None, None], None, dt, tc=tc))
        if m.has_cond:
            for side, stem in (("enc", m.encoder_cond_in), ("dec", m.decoder_cond_in)):
                P[f"{side}_cond_in"] = dict(w=f32(stem[0].weight), b=f32(stem[0].bias))
        q = m.quantizers
        # the reference applies the projections in the module dtype (bf16 weights in bf16 mode)
        P["quant"] = dict(win=q.project_in.weight.detach().to(dt).float().contiguous(), bin=q.project_in.bias.detach().to(dt).float().contiguous(),
                          wout=q.project_out.weight.detach().to(dt).float().contiguous(), bout=q.project_out.bias.detach().to(dt).float().contiguous())
        return P

    # ------------------------------------------------------------------ primitive ops
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, entry, *args, stream=None):
        """Calls launching entry point `entry`(*args, stream) (the current stream by default), raises on its error code and
        adds the kernels it launched, as the library counts them, to `launches`."""
        n0 = self.lib.mv2_launch_count()
        check(getattr(self.lib, entry)(*args, self._stream() if stream is None else stream), entry)
        self.launches += self.lib.mv2_launch_count() - n0

    def _new(self, shape, dtype=None):
        return torch.empty(shape, device=self.device, dtype=dtype or self.dtype)

    def _conv_hist(self, ss: Optional[StreamState], x, need: int):
        """(mv2_conv_hist of the frames in front of x, state update to run after the launch) of a causal conv whose input
        reaches `need` frames back; (None, None) for a whole-clip call.  The history is (buffer, count): a (B, need, ...)
        buffer the stream owns, holding the last `count` frames in front of x at its end (count < need only until the
        stream has seen `need` frames at this layer).  The update keeps its last need frames of [history | x] there."""
        if ss is None or need <= 0:
            return None, None
        h = ss.get("hist")
        hist = None
        if h is not None:
            buf, n = h
            fe = buf[0, 0].numel()
            hist = ConvHist(h=buf.data_ptr() + (need - n) * fe * buf.element_size(), T_h=n, clip_stride=need * fe)

        def advance():
            T = x.shape[1]
            buf, n = h if h is not None else (self._new((x.shape[0], need) + tuple(x.shape[2:]), x.dtype), 0)
            keep = min(T, need)
            old = min(n, need - keep)
            # the older frames move T places towards the front, one frame per copy in increasing order: source and
            # destination ranges overlap when T < old
            for i in range(old):
                self.copy_frames(buf, need - old + i, 1, dst=buf, dst_t0=need - keep - old + i)
            self.copy_frames(x, T - keep, keep, dst=buf, dst_t0=need - keep)
            ss.put("hist", (buf, old + keep))
        return hist, advance

    def _hist_cat(self, ss: StreamState, x):
        """[carried history | x] as one new (B, T_h + T, ...) tensor."""
        buf, n = ss.get("hist")
        cat = self._new((x.shape[0], n + x.shape[1]) + tuple(x.shape[2:]), x.dtype)
        self.copy_frames(buf, buf.shape[1] - n, n, dst=cat, dst_t0=0)
        self.copy_frames(x, 0, x.shape[1], dst=cat, dst_t0=n)
        return cat

    def conv(self, x, pk: ConvPack, *, stride=(1, 1, 1), pad=None, out_spatial=None, act=ACT_NONE,
             res=None, shuffle=SHUFFLE_NONE, token_shift=False, out_cf=False, oscale=None, ss: Optional[StreamState] = None):
        """x: (B,T,H,W,Ci) channels-last.  `pad` = leading (pt,ph,pw); causal default (kt-1, kh//2, kw//2).
        out_cf (wgmma slab path, Co % 8 != 0 only): write torch's (B,Co,To,Ho,Wo) layout directly.
        ss: stream state of this conv -- the frames in front of x are read from the carried history, and the last
        k_t - 1 input frames are kept for the next chunk."""
        B, Ti, Hi, Wi, Ci = x.shape
        hist, advance = self._conv_hist(ss, x, pk.k[0] - 1)
        ta = self._tc_args(x, pk, stride, pad, out_spatial, act, shuffle, out_cf, res=res, oscale=oscale)
        kind = self.conv_kernel(ta, pk, 0 if hist is None else hist.T_h, token_shift)
        To, Ho, Wo = ta.To, ta.Ho, ta.Wo
        if kind == "simt":
            assert Ci == pk.Ci and pk.w is not None and not out_cf, "wgmma-only weight pack or layout has no CUDA-core path"
            co = pk.Co
        else:
            co = pk.Co_tc // 2 if pk.epi_mode == 1 else pk.Co_tc
        if shuffle == SHUFFLE_SPACE:
            y = self._new((B, To, 2 * Ho, 2 * Wo, co // 4))
        elif shuffle == SHUFFLE_TIME:
            y = self._new((B, 2 * To, Ho, Wo, co // 2))
        elif out_cf:
            y = self._new((B, co, To, Ho, Wo))
        else:
            y = self._new((B, To, Ho, Wo, co))
        if res is not None:
            assert res.shape == y.shape and res.dtype == y.dtype and res.is_contiguous()
        hist_p = None if hist is None else C.byref(hist)
        if kind == "simt":
            a = ConvArgs(x=_ptr(x), w=_ptr(pk.w), bias=_ptr(pk.bias), res=_ptr(res), y=_ptr(y), dtype=_dt(self.dtype),
                         B=B, Ti=Ti, Hi=Hi, Wi=Wi, Ci=Ci, To=To, Ho=Ho, Wo=Wo, Co=pk.Co,
                         kt=ta.kt, kh=ta.kh, kw=ta.kw, st=ta.st, sh=ta.sh, sw=ta.sw, pt=ta.pt, ph=ta.ph, pw=ta.pw,
                         act=act, shuffle=shuffle, x_token_shift=int(token_shift), oscale=_ptr(oscale))
            entry, args = "mv2_conv_forward", (C.byref(a), hist_p)
        elif kind == "down":
            ta.y, ta.w = _ptr(y), _ptr(pk.w_down)
            entry, args = "mv2_tc_down_space_forward", (C.byref(ta),)
        else:
            ta.y = _ptr(y)
            if kind == "tap_cat":
                # shapes the history operand does not take (a strided conv, or frame tiles of < 8 positions): the same
                # kernel on a copy of [history | x] with the leading padding shortened by the history, which gives the
                # same products per output element
                cat = self._hist_cat(ss, x)
                ta.x, ta.Ti, ta.pt = _ptr(cat), cat.shape[1], ta.pt - hist.T_h
                kind, hist_p = "tap", None
            entry = "mv2_tc_slab_forward" if kind == "slab" else "mv2_tc_conv_forward"
            args = (C.byref(ta), hist_p)
        self._conv_launch(kind, entry, args, Ci=Ci, Co=co, k=tuple(pk.k), out=(B, To, Ho, Wo), macs=pk.macs, act=act,
                          shuffle=shuffle, res=res is not None, epi_mode=pk.epi_mode, stride=tuple(stride))
        if advance is not None:
            advance()
        if kind == "simt" and pk.epi_mode == 2:   # scaled residual: the residual epilogue, then * 2^-0.5 (the reference's add-then-multiply)
            assert res is not None and shuffle == SHUFFLE_NONE
            scale = torch.full((B, pk.Co), 2 ** -0.5, device=self.device, dtype=torch.float32)
            self._call("mv2_scale_channels", _ptr(y), _ptr(scale), _ptr(y), _dt(self.dtype), B, To * Ho * Wo, pk.Co)
        return y

    def conv_kernel(self, ta: TcConvArgs, pk: ConvPack, hist_T: int = 0, token_shift: bool = False) -> str:
        """The kernel conv() runs for the call `ta` (its mv2_tc_conv_args) with hist_T history frames: "slab" (tc_slab.cu),
        "down" (its SpatialDownsample2x flavour, on pk.w_down), "tap" (tc_conv.cu), "tap_cat" (tc_conv.cu on a copy of
        [history | x]) or "simt" (the CUDA-core conv).  Host-side shape queries only: it launches nothing and needs no device."""
        if not (tensor_core_dtype(self.dtype, self.tf32) and self.use_tc and pk.w_tc is not None and ta.Ci == pk.Ci_tc
                and not token_shift):
            return "simt"
        lib = self.lib
        # the persistent slab kernel reuses each activation slab for all in-plane taps, so it takes every layer it supports
        # (incl. the 64-byte-row conv_in); the tap-wise kernel keeps the strided down-samplers that have no down-space pack.
        # tc_variant = "tap" forces the tap-wise kernel (tests / sweeps).
        if self.tc_variant != "tap":
            if lib.mv2_tc_slab_supported(C.byref(ta)):
                return "slab"
            if pk.w_down is not None and lib.mv2_tc_down_space_supported(C.byref(ta)):
                return "down"
        if not lib.mv2_tc_conv_supported(C.byref(ta)):
            return "simt"
        return "tap_cat" if hist_T > 0 and not lib.mv2_tc_conv_hist_supported(C.byref(ta)) else "tap"

    def _conv_launch(self, kind, entry, args, *, Ci, Co, k, out, macs, act, shuffle=SHUFFLE_NONE, res=False, epi_mode=0,
                     stride=(1, 1, 1), fused_ru=False):
        """Launches conv kernel `entry`(*args, stream) of `kind` ("slab", "down", "tap" or "simt") and accounts for it: the
        counters, CUDA events around it inside profile_convs and, for the tensor-core kernels, a conv_log record.  out:
        (B, To, Ho, Wo) output positions; macs: multiply-accumulates per position.  The down-space kernel is a flavour of the
        slab kernel: it counts, profiles and logs as "slab", and its record has down_space=True."""
        down_space = kind == "down"
        kind = "slab" if down_space else kind
        prof = self._prof is not None and kind != "simt"
        if prof:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        self._call(entry, *args)
        if kind == "simt":
            self.simt_conv_calls += 1
            return
        if prof:
            e1.record()
            self._prof.append((e0, e1, 2.0 * math.prod(out) * macs, kind, math.prod(k)))
        if self.conv_log is not None:
            self.conv_log.append(dict(kind=kind, Ci=Ci, Co=Co, k=k, out=out, geglu=epi_mode == 1, shuffle=shuffle, res=res,
                                      act=act, epi_mode=epi_mode, stride=stride, fused_ru=fused_ru, down_space=down_space))
        self.tc_calls += 1
        self.slab_calls += kind != "tap"
        self.fused_ru_calls += fused_ru

    def _tc_args(self, x, pk: ConvPack, stride=(1, 1, 1), pad=None, out_spatial=None, act=ACT_NONE, shuffle=SHUFFLE_NONE,
                 out_cf=False, res=None, y=None, oscale=None):
        """The mv2_tc_conv_args of conv(x, pk, ...) on the wgmma kernels, with conv's defaults for pad and out_spatial.  x may
        be the input's shape instead, for a conv_kernel query before the input exists."""
        B, Ti, Hi, Wi, Ci = x.shape if isinstance(x, torch.Tensor) else x
        kt, kh, kw = pk.k_tc or pk.k
        pt, ph, pw = (kt - 1, kh // 2, kw // 2) if pad is None else pad
        To, Ho, Wo = (Ti, Hi, Wi) if out_spatial is None else out_spatial
        return TcConvArgs(x=_ptr(x) if isinstance(x, torch.Tensor) else None, w=_ptr(pk.w_tc), bias=_ptr(pk.bias_tc),
                          res=_ptr(res), y=_ptr(y), B=B, Ti=Ti, Hi=Hi, Wi=Wi, Ci=Ci, To=To, Ho=Ho, Wo=Wo, Co=pk.Co_tc,
                          kt=kt, kh=kh, kw=kw, st=stride[0], sh=stride[1], sw=stride[2],
                          pt=pt, ph=ph, pw=pw, act=act, shuffle=shuffle, epi_mode=pk.epi_mode,
                          oscale=_ptr(oscale), out_layout=int(out_cf), dtype=self._tc_dt())

    def _tc_dt(self) -> int:
        """Element type of this engine's wgmma launches (mv2_tc_conv_args.dtype): fp32 storage is MV2_TF32."""
        return MV2_TF32 if self.dtype == torch.float32 else _dt(self.dtype)

    def conv_cf_supported(self, x, pk: ConvPack, pad, out_spatial) -> bool:
        """True when conv(x, pk, pad=pad, out_spatial=out_spatial, out_cf=True) runs: bf16 / fp16 on the slab kernel, whose
        channels-first epilogue takes fewer than 8 (or a ragged number of) output channels."""
        return self.conv_kernel(self._tc_args(x, pk, pad=pad, out_spatial=out_spatial, out_cf=True), pk) == "slab"

    def residual_unit(self, x, p, ss: Optional[StreamState] = None):
        """ResidualUnit (reference M:930-944): x + SE(ELU(conv1(ELU(causal_conv3(x)))))."""
        B, T, H, W, Cc = x.shape
        F_, Pn = B * T, H * W
        dt = _dt(self.dtype)
        c3, c1 = p["conv3"], p["conv1"]
        if self.fuse_ru and self.conv_kernel(self._tc_args(x, c3, act=ACT_ELU), c3) == "slab":
            ra = TcRuArgs(x=_ptr(x), w3=_ptr(c3.w_tc), b3=_ptr(c3.bias_tc), w1=_ptr(c1.w_tc), b1=_ptr(c1.bias_tc),
                          se_wk=_ptr(p["wk"]), se_bk=p["bk"], y=None, se_ws=None, B=B, T=T, H=H, W=W, C=Cc,
                          kt=c3.k[0], kh=c3.k[1], kw=c3.k[2], dtype=self._tc_dt())
            if self.lib.mv2_tc_ru_supported(C.byref(ra)):
                hist, advance = self._conv_hist(_sub(ss, "conv3"), x, c3.k[0] - 1)
                y = self._new(x.shape)
                ws = self._new((self.lib.mv2_tc_ru_workspace_bytes(C.byref(ra)) // 4,), torch.float32)
                ra.y, ra.se_ws = _ptr(y), _ptr(ws)
                nrec = self.lib.mv2_tc_ru_records(C.byref(ra))
                self._conv_launch("slab", "mv2_tc_ru_forward", (C.byref(ra), None if hist is None else C.byref(hist)), Ci=Cc,
                                  Co=Cc, k=tuple(c3.k), out=(B, T, H, W), macs=c3.macs + c1.macs, act=ACT_ELU, fused_ru=True)
                if advance is not None:
                    advance()
                gates = self._new((F_, Cc), torch.float32)
                self._call("mv2_se_gate_records", _ptr(ws), nrec, F_, Cc, p["hidden"], _ptr(p["w1"]), _ptr(p["b1"]), _ptr(p["w2"]),
                           _ptr(p["b2"]), _ptr(gates))
                out = self._new(x.shape)
                self._call("mv2_gate_residual", _ptr(y), _ptr(x), _ptr(gates), _ptr(out), dt, F_, Pn, Cc)
                return out
        h = self.conv(x, c3, act=ACT_ELU, ss=_sub(ss, "conv3"))
        y = self.conv(h, c1, act=ACT_ELU)
        return self.squeeze_excite_residual(y, x, p)

    def squeeze_excite_residual(self, y, x, p):
        """x + SqueezeExcite(y) (M:221-240) of an unfused ResidualUnit: softmax pool of y per frame, gate MLP, gated residual."""
        B, T, H, W, Cc = x.shape
        F_, Pn = B * T, H * W
        dt = _dt(self.dtype)
        ws = self._new((self.lib.mv2_se_workspace_bytes(F_, Pn, Cc) // 4,), torch.float32)
        gates = self._new((F_, Cc), torch.float32)
        self._call("mv2_se_pool", _ptr(y), dt, F_, Pn, Cc, _ptr(p["wk"]), p["bk"], _ptr(ws))
        self._call("mv2_se_gate", _ptr(ws), dt, F_, Pn, Cc, p["hidden"], _ptr(p["w1"]), _ptr(p["b1"]), _ptr(p["w2"]),
                   _ptr(p["b2"]), _ptr(gates))
        out = self._new(x.shape)
        self._call("mv2_gate_residual", _ptr(y), _ptr(x), _ptr(gates), _ptr(out), dt, F_, Pn, Cc)
        return out

    def dense_small(self, x, w, b, act=ACT_NONE):
        """fp32 y[b][n] = act(x[b] . w[n] + bias[n]) (cond stems M:1344-1352, to_cond M:983)."""
        Bx, K = x.shape
        N = w.shape[0]
        y = self._new((Bx, N), torch.float32)
        self._call("mv2_dense_small", _ptr(x), _ptr(w), _ptr(b), _ptr(y), Bx, K, N, act)
        return y

    def cond_stem(self, cond, side):
        p = self._packs[f"{side}_cond_in"]
        return self.dense_small(cond.float().contiguous(), p["w"], p["b"], ACT_SILU)

    def residual_unit_mod(self, x, p, cond_e, ss: Optional[StreamState] = None):
        """ResidualUnitMod (M:978-988): x + ELU(conv_out(ELU(Conv3DMod(x, to_cond(cond))))).  The per-clip modulated weights
        are never built: input channels are scaled by (cond + 1), the shared-weight conv runs unchanged and the demodulation
        rsqrt(sum w_b^2) multiplies the accumulator per (clip, output channel) in the epilogue (include/magvit2_b200.h)."""
        B, T, H, W, Cc = x.shape
        c = self.dense_small(cond_e, p["wc"], p["bc"])
        scale_in = self._new((B, Cc), torch.float32)
        inv_norm = self._new((B, Cc), torch.float32)
        self._call("mv2_mod_prepare", _ptr(c), _ptr(p["S"]), p["eps"], _ptr(scale_in), _ptr(inv_norm), B, Cc, Cc)
        xs = self._new(x.shape)
        self._call("mv2_scale_channels", _ptr(x), _ptr(scale_in), _ptr(xs), _dt(self.dtype), B, T * H * W, Cc)
        h = self.conv(xs, p["conv3"], act=ACT_ELU, oscale=inv_norm, ss=_sub(ss, "conv3"))
        return self.conv(h, p["conv1"], act=ACT_ELU, res=x)

    def rmsnorm(self, x, gamma, token_shift=False, ss: Optional[StreamState] = None):
        """ss (token shift only): the shifted channels of frame 0 come from the previous chunk's last frame, which the
        stream keeps in a (B, 1, ...) buffer of its own."""
        B, T, H, W, Cc = x.shape
        out = self._new(x.shape)
        prev = None if (ss is None or not token_shift) else ss.get("prev")
        if prev is not None:
            self._call("mv2_rmsnorm_prev", _ptr(x), _ptr(prev), prev[0, 0].numel(), _ptr(out), _dt(self.dtype), _ptr(gamma),
                       B, T, H * W, Cc)
        else:
            self._call("mv2_rmsnorm", _ptr(x), _ptr(out), _dt(self.dtype), _ptr(gamma), B, T, H * W, Cc, int(token_shift))
        if ss is not None and token_shift:
            if prev is None:
                prev = self._new((B, 1, H, W, Cc), x.dtype)
                ss.put("prev", prev)
            self.copy_frames(x, T - 1, 1, dst=prev)
        return out

    def feed_forward(self, x, p, token_shift=False, ss: Optional[StreamState] = None):
        """Residual(FeedForward) (M:471-508, M:1191): x + fc2(geglu(fc1(rmsnorm(shift(x)))))."""
        B, T, H, W, Cc = x.shape
        xn = self.rmsnorm(x, p["gamma"], token_shift, ss)
        fc1 = p["fc1"]
        if self.conv_kernel(self._tc_args(xn, fc1), fc1) != "simt":
            g = self.conv(xn, fc1)                            # fc1 + bias + GEGLU fused, hidden width padded to 64
            return self.conv(g, p["fc2"], res=x)
        hdn = self.conv(xn, fc1)
        I = p["inner"]
        g = self._new((B, T, H, W, I))
        self._call("mv2_geglu", _ptr(hdn), _ptr(g), _dt(self.dtype), B * T * H * W, I)
        return self.conv(g, p["fc2"], res=x)

    def attention(self, x, p, axis: str, dropout: Optional[_lib.DropoutArgs] = None, ss: Optional[StreamState] = None):
        """Residual(SpaceAttention) / Residual(TokenShift(TimeAttention)) (M:444-464, M:1190, M:1235).  `dropout`: drop the
        softmax weights with that (seed, call, p) mask (Attend in training mode, A:175 / A:239)."""
        B, T, H, W, Cc = x.shape
        time_axis = axis == "time"
        xn = self.rmsnorm(x, p["gamma"], token_shift=time_axis, ss=ss)
        qkv = self.conv(xn, p["qkv"])
        if time_axis and ss is not None:
            step = lambda: self._attention_tail(qkv, p, ss)     # noqa: E731
            o = step() if self.host_step is None else self.host_step(step)
            return self.conv(o, p["out"], res=x)
        heads, dh = p["heads"], p["dim_head"]
        o = self._new((B, T, H, W, heads * dh))
        HW = H * W
        if time_axis:
            a = AttnArgs(qkv=_ptr(qkv), out=_ptr(o), mem_kv=_ptr(p["mem_kv"]), dtype=_dt(self.dtype), heads=heads,
                         dim_head=dh, n_mem=p["n_mem"], causal=1, n_outer=B, n_inner=HW, L=T,
                         outer_stride=T * HW, inner_stride=1, tok_stride=HW)
        else:
            a = AttnArgs(qkv=_ptr(qkv), out=_ptr(o), mem_kv=_ptr(p["mem_kv"]), dtype=_dt(self.dtype), heads=heads,
                         dim_head=dh, n_mem=p["n_mem"], causal=0, n_outer=B * T, n_inner=1, L=HW,
                         outer_stride=HW, inner_stride=0, tok_stride=1)
        if dropout is None:
            self._call("mv2_attention", C.byref(a))
        else:
            self._call("mv2_attention_dropout", C.byref(a), C.byref(dropout))
        return self.conv(o, p["out"], res=x)

    KV_CACHE_STEP = 16       # latent frames the time attention's K/V cache grows by

    def _attention_tail(self, qkv, p, ss: StreamState):
        """Time attention of a streamed chunk -> its output o, a buffer the stream keeps per chunk length: the chunk's keys
        and values are appended to the stream's K/V cache (every earlier frame's; it grows by KV_CACHE_STEP frames when
        full) and mv2_attention_tail computes the chunk's queries, read from qkv, against all cached keys.  Its launch
        arguments change with every push (the cache length, the kernel chosen for it, the cache's address after a growth),
        so a captured push runs it as a host step between two graph segments (host_step).

        The cache has one time axis for all rows, and each row's clip starts at its own index of it (StreamState.restart_rows;
        0 for a row never restarted).  Each run of consecutive rows that share a start gets its own call on the cache from
        that start, so every row sees its own clip's keys with the kernel chosen for their count, as in a new stream.  When
        the cache grows, the frames before the earliest start are dropped (kv_cache_plan)."""
        B, T, H, W, C3 = qkv.shape
        HW, HD = H * W, C3 // 3
        outs = ss.get("o")
        if outs is None:
            outs = {}
            ss.put("o", outs)
        o = outs.get(T)
        if o is None:
            o = outs[T] = self._new((B, T, H, W, HD))
        buf, L0, starts = ss.get("kv") or (None, 0, (0,) * B)
        if buf is None or buf.shape[1] < L0 + T:
            drop, cap = kv_cache_plan(L0, T, starts, self.KV_CACHE_STEP)
            nbuf = self._new((B, cap, H, W, 2 * HD))
            if L0 > drop:
                self.copy_frames(buf, drop, L0 - drop, dst=nbuf, dst_t0=0)
            buf, L0, starts = nbuf, L0 - drop, tuple(s - drop for s in starts)
        buf[:, L0:L0 + T].copy_(qkv[..., HD:])           # the '(kv h d)' two thirds of each '(qkv h d)' row
        L = L0 + T
        ss.put("kv", (buf, L, starts))
        cap, es = buf.shape[1], buf.element_size()
        for r0, r1, s in row_runs(starts):
            a = AttnArgs(qkv=_ptr(buf) + (r0 * cap + s) * HW * 2 * HD * es, out=None, mem_kv=_ptr(p["mem_kv"]),
                         dtype=_dt(self.dtype), heads=p["heads"], dim_head=p["dim_head"], n_mem=p["n_mem"], causal=1,
                         n_outer=r1 - r0, n_inner=HW, L=L - s, outer_stride=cap * HW, inner_stride=1, tok_stride=HW)
            self._call("mv2_attention_tail", C.byref(a), _ptr(qkv) + r0 * T * HW * C3 * es, T * HW, L0 - s,
                       _ptr(o) + r0 * T * HW * HD * es, T * HW)
        return o

    def attention_dropout_mask(self, n_seq, heads, L, n_mem, dropout: _lib.DropoutArgs):
        """The keep mask of an attention call, uint8 (n_seq, heads, L, n_mem + L) (mv2_attention_dropout_mask)."""
        keep = torch.empty((n_seq, heads, L, n_mem + L), device=self.device, dtype=torch.uint8)
        self._call("mv2_attention_dropout_mask", n_seq, heads, L, n_mem, C.byref(dropout), _ptr(keep))
        return keep

    def linear_attention(self, x, p):
        """Residual(LinearSpaceAttention) (M:421-442, M:1207)."""
        B, T, H, W, Cc = x.shape
        xn = self.rmsnorm(x, p["gamma"])
        q = self.conv(xn, p["q"])
        kv = self.conv(xn, p["kv"])
        heads, dh = p["heads"], p["dim_head"]
        n_seq, L = B * T, H * W
        ws = self._new((self.lib.mv2_linattn_workspace_bytes(n_seq, heads, L) // 4,), torch.float32)
        o = self._new((B, T, H, W, heads * dh))
        self._call("mv2_linear_attention", _ptr(q), _ptr(kv), _ptr(o), _dt(self.dtype), n_seq, L, heads, dh, _ptr(ws))
        return self.conv(o, p["out"], res=x)

    def gateloop(self, x, p, ss: Optional[StreamState] = None):
        """ToTimeSequence(Residual(SimpleGateLoopLayer)) (M:178-191, M:1216-1222): RMSNorm, Linear(dim, 3 dim), then the gated
        recurrence over time per (pixel, channel) with the residual add fused (mv2_gateloop_scan)."""
        B, T, H, W, Cc = x.shape
        qkva = self.conv(self.rmsnorm(x, p["gamma"]), p["qkva"])
        out = self._new(x.shape)
        if ss is not None:            # the fp32 scan state s_{t-1} per (clip, pixel, channel) carries over to the next chunk
            state = ss.get("s")
            if state is None:
                state = torch.zeros((B, H * W, Cc), device=self.device, dtype=torch.float32)
                ss.put("s", state)
            self._call("mv2_gateloop_scan_state", _ptr(qkva), _ptr(x), _ptr(out), _dt(self.dtype), B, T, H * W, Cc, _ptr(state))
        else:
            self._call("mv2_gateloop_scan", _ptr(qkva), _ptr(x), _ptr(out), _dt(self.dtype), B, T, H * W, Cc)
        return out

    def profile_convs(self, fn, steps: int = 3):
        """Runs fn() `steps` times with CUDA events around every wgmma conv launch (on the launching stream).
        A long spin kernel is queued first so the host runs ahead of the GPU and the event pairs bracket pure
        kernel time, not host launch gaps.  Returns {class: (kernel ms per step, launches per step, FLOPs per step)}
        for class in 'conv3d' (taps > 1 convs in tc_slab_kernel: the causal Conv3d path) and 'all' (every wgmma launch)."""
        fn()
        torch.cuda.synchronize(self.device)
        self._prof = []
        try:
            for _ in range(steps):
                torch.cuda._sleep(int(40e6))          # ~20 ms of GPU busy-wait: lets the host enqueue the whole step
                fn()
            torch.cuda.synchronize(self.device)
            recs = [(e0.elapsed_time(e1), f, kind, taps) for e0, e1, f, kind, taps in self._prof]
        finally:
            self._prof = None
        out = {}
        for name, sel in (("conv3d", lambda r: r[2] == "slab" and r[3] > 1), ("all", lambda r: True)):
            rs = [r for r in recs if sel(r)]
            if rs:
                out[name] = (sum(r[0] for r in rs) / steps, len(rs) // steps, sum(r[1] for r in rs) / steps)
        return out

    # ------------------------------------------------------------------ stages
    def _stage(self, x, st, key, decoder: bool, cond_e=None, ss: Optional[StreamState] = None):
        P = self._packs
        B, T, H, W, Cc = x.shape
        if st.kind == "residual":
            for j in range(st.count):
                x = self.residual_unit(x, P[f"{key}.{j}"], _sub(ss, str(j)))
        elif st.kind == "cond_residual":
            x = self.residual_unit_mod(x, P[key], cond_e, ss)
        elif st.kind == "compress_space":
            if decoder:   # SpatialUpsample2x (M:838-846)
                x = self.conv(x, P[key], act=ACT_SILU, shuffle=SHUFFLE_SPACE)
            else:         # SpatialDownsample2x (M:770-780): Conv2d k3 s2 p1
                x = self.conv(x, P[key], stride=(1, 2, 2), pad=(0, 1, 1),
                              out_spatial=(T, (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1))
        elif st.kind == "compress_time":
            if decoder:   # TimeUpsample2x (M:875-883)
                x = self.conv(x, P[key], act=ACT_SILU, shuffle=SHUFFLE_TIME)
            else:         # TimeDownsample2x (M:796-807): pad (2, 0), Conv1d k3 s2
                x = self.conv(x, P[key], stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=((T + 2 - 3) // 2 + 1, H, W), ss=ss)
        elif st.kind in ("attend_space", "attend_time"):
            time_axis = st.kind == "attend_time"
            drop = () if self.dropout is None else (self.dropout.take(),)      # without dropout: the plain call
            if time_axis and ss is not None:
                x = self.attention(x, P[key + ".attn"], "time", ss=ss.sub("attn"))
                x = self.feed_forward(x, P[key + ".ff"], token_shift=True, ss=ss.sub("ff"))
            else:
                x = self.attention(x, P[key + ".attn"], "time" if time_axis else "space", *drop)
                x = self.feed_forward(x, P[key + ".ff"], token_shift=time_axis)
        elif st.kind == "linear_attend_space":
            x = self.linear_attention(x, P[key + ".attn"])
            x = self.feed_forward(x, P[key + ".ff"])
        elif st.kind == "gateloop_time":
            x = self.gateloop(x, P[key], ss)
        else:
            raise ValueError(st.kind)
        return x

    def _tap(self, name, x):
        if self.taps is not None:
            self.taps[name] = x.permute(0, 4, 1, 2, 3).float().cpu()

    # ------------------------------------------------------------------ layout
    def to_channels_last(self, v: torch.Tensor, t_pad: int = 0):
        """(B,C,T,H,W) torch tensor (fp32, bf16, or uint8 frames: normalised x / 255 as the reference's data loaders do,
        D:103, D:188) -> (B,T+t_pad,H,W,C) compute dtype."""
        if v.dtype not in self._src_dtypes():
            v = v.float()
        v = v.contiguous()
        B, Cc, T, H, W = v.shape
        out = self._new((B, T + t_pad, H, W, Cc))
        self._call("mv2_to_channels_last", _ptr(v), _src_dt(v.dtype), _ptr(out), _dt(self.dtype), B, Cc, T, H, W, t_pad)
        return out

    def _src_dtypes(self):
        """Video dtypes the layout-in kernels read directly (others are converted to fp32 first)."""
        return (torch.float32, torch.bfloat16, torch.uint8) + ((torch.float16,) if self.dtype == torch.float16 else ())

    def ingest_kwpack(self, v: torch.Tensor, t_pad: int, pin):
        """(B,C,T,H,W) -> (B,T+t_pad,H,W,32) with the k_w taps packed into channels (mv2_ingest_kwpack), in the compute
        dtype: mv2_ingest_kwpack writes fp16 for an fp16 source and bf16 for the others, so an fp16 model's uint8 / fp32
        video is first rounded to fp16 in place of layout (mv2_to_channels_last of single-channel frames: a plain copy);
        an fp32 model's (the TF32 conv_in) is written in fp32 (MV2_KWPACK_F32_DST)."""
        if v.dtype not in self._src_dtypes():
            v = v.float()
        v = v.contiguous()
        B, Cc, T, H, W = v.shape
        if self.dtype == torch.float16 and v.dtype != torch.float16:
            v16 = self._new(tuple(v.shape), torch.float16)
            self._call("mv2_to_channels_last", _ptr(v), _src_dt(v.dtype), _ptr(v16), MV2_F16, B * Cc * T, 1, 1, H, W, 0)
            v = v16
        out = self._new((B, T + t_pad, H, W, pin.Ci_tc), self.dtype)
        dst32 = _lib.MV2_KWPACK_F32_DST if self.dtype == torch.float32 else 0
        self._call("mv2_ingest_kwpack", _ptr(v), _src_dt(v.dtype) | dst32, _ptr(out), B, Cc, T, H, W, t_pad, pin.kw_orig,
                   pin.kw_orig // 2, pin.Ci_tc)
        return out

    _PAD_MODES = {"reflect": 1, "replicate": 2, "circular": 3}

    def causal_conv_padded(self, x, pk, pad_mode):
        """CausalConv3d with pad_mode != 'constant' (M:925-927): the padding is materialised by mv2_pad_cl, then the conv
        runs without any implicit padding.  As in the reference the mode falls back to 'constant' when time_pad >= T."""
        B, T, H, W, Cc = x.shape
        kt, kh, kw = pk.k
        if pad_mode == "constant" or kt - 1 >= T:
            return self.conv(x, pk)
        xp = self._new((B, T + kt - 1, H + 2 * (kh // 2), W + 2 * (kw // 2), Cc))
        self._call("mv2_pad_cl", _ptr(x), _ptr(xp), _dt(self.dtype), B, T, H, W, Cc, kt - 1, kh // 2, kw // 2,
                   self._PAD_MODES[pad_mode])
        return self.conv(xp, pk, pad=(0, 0, 0), out_spatial=(T, H, W))

    def copy_frames(self, src, t0, n, dst=None, dst_t0=0, zero_front=False):
        """Frames [t0, t0 + n) of a channels-last clip tensor -> a new (B, n, ...) tensor, or into ``dst`` at ``dst_t0``."""
        B, Ts = src.shape[:2]
        if dst is None:
            dst = self._new((B, n) + tuple(src.shape[2:]), src.dtype)
        frame_bytes = src[0, 0].numel() * src.element_size()
        assert dst[0, 0].numel() * dst.element_size() == frame_bytes and src.is_contiguous() and dst.is_contiguous()
        self._call("mv2_copy_frames", _ptr(src), _ptr(dst), B, Ts, dst.shape[1], t0, dst_t0, n, frame_bytes, int(zero_front))
        return dst

    def to_channels_first(self, x: torch.Tensor, t_crop: int = 0, out_dtype=None):
        B, T, H, W, Cc = x.shape
        out_dtype = out_dtype or self.dtype
        out = torch.empty((B, Cc, T - t_crop, H, W), device=self.device, dtype=out_dtype)
        self._call("mv2_to_channels_first", _ptr(x), _dt(x.dtype), _ptr(out), _dt(out_dtype), B, Cc, T, H, W, t_crop)
        return out

    def mse(self, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        """F.mse_loss(a, b) of two same-layout tensors (reference M:1722: video vs reconstruction, both (B,C,T,H,W)) as a 0-d
        fp32 tensor; `a` may hold uint8 frames (x / 255)."""
        assert a.shape == b.shape, (a.shape, b.shape)
        if a.dtype not in self._src_dtypes():
            a = a.float()
        a, b = a.contiguous(), b.contiguous()
        ws = self._new((self.lib.mv2_mse_workspace_bytes() // 4,), torch.float32)
        out = self._new((1,), torch.float32)
        self._call("mv2_mse", _ptr(a), _src_dt(a.dtype), _ptr(b), _dt(b.dtype), a.numel(), _ptr(ws), _ptr(out))
        return out[0]

    def maxpool2x2(self, x):
        """nn.MaxPool2d(2, 2) (floor mode) of a channels-last (B, T, H, W, C) map -> (B, T, H // 2, W // 2, C)."""
        B, T, H, W, Cc = x.shape
        y = self._new((B, T, H // 2, W // 2, Cc), x.dtype)
        self._call("mv2_maxpool2x2", _ptr(x), _ptr(y), _dt(x.dtype), B * T, H, W, Cc)
        return y

    def maxpool2x2_backward(self, g, x):
        """Gradient wrt the pool's input x (the output of a conv with ReLU in its epilogue) from the pool output's gradient g:
        each window's gradient goes to its first maximum, masked by x > 0; dense (B, T, H, W, C)."""
        B, T, H, W, Cc = x.shape
        g = g.to(x.dtype).contiguous()
        assert tuple(g.shape) == (B, T, H // 2, W // 2, Cc), (g.shape, x.shape)
        gx = self._new(x.shape, x.dtype)
        self._call("mv2_maxpool2x2_backward", _ptr(g), _ptr(x), _ptr(gx), _dt(x.dtype), B * T, H, W, Cc)
        return gx

    # ------------------------------------------------------------------ the path
    def conv_in(self, video: torch.Tensor, first_frame: bool = True, ss: Optional[StreamState] = None, sff_rest: bool = False):
        """video (B,C,T,H,W) on device -> conv_in's output (B,T+t_pad,H,W,C) channels-last.  The time_padding zero frames
        are only prepended when the clip starts with a first frame (video_contains_first_frame, M:1534-1537).
        sff_rest: a streamed chunk after the first frame of a separate_first_frame_encoding clip (the causal conv_in of
        frames 1.., which the whole-clip call runs on channels-last frames)."""
        m = self.model
        t_pad = m.time_padding if first_frame else 0
        pin = self._packs.get("conv_in_tc")
        ss = _sub(ss, "conv_in")
        B, _, T, H, W = video.shape
        if sff_rest:
            x = self.conv(self.to_channels_last(video, 0), self._packs["conv_in"], ss=ss)
        elif m.separate_first_frame_encoding and first_frame:
            # M:1553-1561: the first frame goes through its own 2-D conv, frames 1.. through the causal conv_in on their own,
            # then the feature map is [time_padding zero frames, first, rest]
            v_cl = self.to_channels_last(video, 0)
            parts = [(self.conv(self.copy_frames(v_cl, 0, 1), self._packs["conv_in_ff"]), t_pad)]
            if T > 1:
                rest = self.copy_frames(v_cl, 1, T - 1)
                parts.append((self.conv(rest, self._packs["conv_in"], ss=ss) if ss is not None else
                              self.causal_conv_padded(rest, self._packs["conv_in"], m.conv_in.pad_mode), t_pad + 1))
            x = self._new((B, T + t_pad, H, W, parts[0][0].shape[-1]))
            for i, (part, t0) in enumerate(parts):
                self.copy_frames(part, 0, part.shape[1], dst=x, dst_t0=t0, zero_front=(i == 0))
        elif m.conv_in.pad_mode != "constant":
            x = self.causal_conv_padded(self.to_channels_last(video, t_pad), self._packs["conv_in"], m.conv_in.pad_mode)
        elif pin is not None and self.conv_kernel(self._tc_args((B, T + t_pad, H, W, pin.Ci_tc), pin), pin) != "simt":
            x = self.ingest_kwpack(video, t_pad, pin)
            x = self.conv(x, pin, pad=(pin.k_tc[0] - 1, pin.k_tc[1] // 2, 0), ss=ss)
        else:
            x = self.to_channels_last(video, t_pad)
            x = self.conv(x, self._packs["conv_in"], ss=ss)
        return x

    def encode_cl(self, video: torch.Tensor, first_frame: bool = True, cond=None, ss: Optional[StreamState] = None,
                  sff_rest: bool = False):
        """video (B,C,T,H,W) on device -> encoder output, channels-last.  Reference encode M:1523-1576.  ss / sff_rest:
        one chunk of a streamed clip (stream.TokenizeStream)."""
        m = self.model
        x = self.conv_in(video, first_frame, ss, sff_rest)
        self._tap("conv_in", x)
        cond_e = self.cond_stem(cond, "enc") if (m.has_cond and cond is not None) else None     # M:1544-1548
        for i, st in enumerate(m.stages):
            x = self._stage(x, st, f"enc{i}", decoder=False, cond_e=cond_e, ss=_sub(ss, f"enc{i}"))
            self._tap(f"enc{i}", x)
        return x

    def decode_cl(self, q: torch.Tensor, first_frame: bool = True, cond=None, ss: Optional[StreamState] = None,
                  sff_rest: bool = False):
        """quantized channels-last (B,T',H',W',C) -> video (B,3,T,H,W).  Reference decode M:1598-1649.  ss / sff_rest: one
        chunk of a streamed clip (stream.DecodeStream)."""
        m = self.model
        x = q
        cond_e = self.cond_stem(cond, "dec") if (m.has_cond and cond is not None) else None     # M:1612-1616
        for j, st in enumerate(reversed(m.stages)):
            x = self._stage(x, st, f"dec{j}", decoder=True, cond_e=cond_e, ss=_sub(ss, f"dec{j}"))
            self._tap(f"dec{j}", x)
        return self.conv_out(x, first_frame, ss, sff_rest)

    def conv_out(self, x: torch.Tensor, first_frame: bool = True, ss: Optional[StreamState] = None, sff_rest: bool = False):
        """decoder output (B,T,H,W,C) channels-last -> reconstruction (B,3,T-t_pad,H,W).  The leading time_padding frames
        are dropped only for clips that contain a first frame (M:1646-1647).  sff_rest as in conv_in."""
        m = self.model
        pk = self._packs["conv_out"]
        B, T, H, W, Cc = x.shape
        tp = m.time_padding if first_frame else 0
        ss = _sub(ss, "conv_out")
        if sff_rest:
            return self.to_channels_first(self.conv(x, pk, ss=ss))
        if m.separate_first_frame_encoding and first_frame:
            # M:1633-1639: conv_out_first_frame on frame `tp`, the causal conv_out on the frames after it, re-attached
            first = self.conv(self.copy_frames(x, tp, 1), self._packs["conv_out_ff"])
            out = self._new((B, T - tp, H, W, first.shape[-1]))
            self.copy_frames(first, 0, 1, dst=out, dst_t0=0)
            if T - tp > 1:
                rest = self.copy_frames(x, tp + 1, T - tp - 1)
                rest = self.conv(rest, pk, ss=ss) if ss is not None else self.causal_conv_padded(rest, pk, m.conv_out.pad_mode)
                self.copy_frames(rest, 0, T - tp - 1, dst=out, dst_t0=1)
            return self.to_channels_first(out)
        if m.conv_out.pad_mode != "constant":
            return self.to_channels_first(self.causal_conv_padded(x, pk, m.conv_out.pad_mode), t_crop=tp)
        # conv_out writes the reconstruction in torch's (B,C,T,H,W) layout itself and never computes the time_padding frames
        # the reference drops afterwards (M:1642-1647)
        pad, out_sp = (pk.k[0] - 1 - tp, pk.k[1] // 2, pk.k[2] // 2), (T - tp, H, W)
        if (pk.k[2] <= 3            # wider in-plane taps would take the narrow N tiles, which are meant for the video's data gradient
                and Cc % 64 == 0    # 128-byte rows only: a kw = 1 conv_out on 32-channel rows keeps the channels-last conv
                and T > tp and self.conv_cf_supported(x, pk, pad, out_sp)):
            return self.conv(x, pk, pad=pad, out_spatial=out_sp, out_cf=True, ss=ss)
        x = self.conv(x, pk, ss=ss)
        return self.to_channels_first(x, t_crop=tp)

    def quantize_cl(self, x, want_quantized=True, want_aux=False):
        """x channels-last -> (quantized channels-last | None, indices (B,T,H,W[,num_codebooks]), aux fp32 [N][D] | None)."""
        m = self.model
        B, T, H, W, Cc = x.shape
        N = B * T * H * W
        P = self._packs["quant"]
        q = self._new(x.shape) if want_quantized else None
        qz = m.quantizers
        d, nc = qz.codebook_dim, qz.num_codebooks
        ishape = (B, T, H, W) if nc == 1 else (B, T, H, W, nc)      # keep_num_codebooks_dim = num_codebooks > 1 (A.1 step 9)
        aux = self._new((N, d * nc), torch.float32) if want_aux else None
        if m.use_fsq:
            idx = torch.empty(ishape, device=self.device, dtype=torch.int32)
            lv = (C.c_int32 * d)(*qz.levels)
            self._call("mv2_fsq_forward", _ptr(x), _dt(self.dtype), N, Cc, d, nc, lv, _ptr(P["win"]), _ptr(P["bin"]),
                       _ptr(P["wout"]), _ptr(P["bout"]), _ptr(idx), _ptr(q), _ptr(aux))
        else:
            idx = torch.empty(ishape, device=self.device, dtype=torch.int64)
            clamp = qz.soft_clamp_input_value
            self._call("mv2_lfq_forward", _ptr(x), _dt(self.dtype), N, Cc, d, nc, _ptr(P["win"]), _ptr(P["bin"]),
                       _ptr(P["wout"]), _ptr(P["bout"]), float(clamp) if clamp else 0.0, int(qz.spherical),
                       _ptr(idx), _ptr(q), _ptr(aux))
        return q, idx, aux

    def codes_to_quantized_cl(self, codes: torch.Tensor):
        """indices (B,T,H,W[,num_codebooks]) int64/int32 -> quantized channels-last.  LFQ/FSQ.indices_to_codes (M:1593)."""
        m = self.model
        codes = codes.contiguous()
        B, T, H, W = codes.shape[:4]
        qz = m.quantizers
        Cc = qz.dim
        N = B * T * H * W
        P = self._packs["quant"]
        d, nc = qz.codebook_dim, qz.num_codebooks
        q = self._new((B, T, H, W, Cc))
        is64 = int(codes.dtype == torch.int64)
        if m.use_fsq:
            lv = (C.c_int32 * d)(*qz.levels)
            self._call("mv2_fsq_decode", _ptr(codes), is64, N, Cc, d, nc, lv, _ptr(P["wout"]), _ptr(P["bout"]), _ptr(q),
                       _dt(self.dtype))
        else:
            self._call("mv2_lfq_decode", _ptr(codes), is64, N, Cc, d, nc, _ptr(P["wout"]), _ptr(P["bout"]), _ptr(q),
                       _dt(self.dtype))
        return q
