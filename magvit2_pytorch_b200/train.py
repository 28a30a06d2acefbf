"""Training-mode forward with gradients (SURVEY.md 8f N2, first slice): ``model.train(); loss, breakdown =
model(video, return_loss=True); loss.backward()`` for tokenizers without the GAN / perceptual branches
(``use_gan=False, perceptual_loss_weight=0``) -- what ``VideoTokenizerTrainer.train_step`` does with the generator loss
(reference trainer.py:356-363).

Division of labour
  * FORWARD: the hand-written sm_90a kernels of the inference path (engine.Engine / libmagvit2_b200.so), with the
    ResidualUnit run unfused so that its intermediate activations exist.  The activations the backward needs are kept as
    they come out of the kernels (channels-last).
  * BACKWARD: the DATA gradient of the stride-1 causal convs (the 3x3x3 and 1x1x1 convs of every ResidualUnit, conv_out: about
    half of the backward's conv FLOPs) runs on the engine's own conv kernels -- a transposed conv is the same implicit GEMM with
    flipped / transposed weights.  The weight / bias gradients of all convs and the strided down-samplers call
    ``aten.convolution_backward`` (cuDNN) directly on the saved activations -- no forward recomputation.  The light blocks (SqueezeExcite gating, attention / linear-attention /
    FeedForward blocks, the two up-samplers, the quantiser with its straight-through estimator and auxiliary losses) are
    differentiated by re-evaluating a torch restatement of the block on its saved input (``_vjp``).
  There are no dedicated backward kernels (wgrad, attention backward) yet; this slice makes the drop-in claim true for the trainer's generator step,
  it is not a speed claim for training.
The forward is built from three pieces that each record their tape entries -- encoder (conv_in + stages), quantiser, decoder
(stages + conv_out) -- which the training step chains whole and the differentiable encode / decode / decode_from_code_indices
entry points chain in part (DESIGN.md 3.8), all under one autograd.Function (_TapeFn).  Those entry points also need the
gradient wrt their inputs: the cond vector (through the cond stems) and the video, whose data gradient through conv_in runs on
the slab kernel's narrow N tile in bf16 and on the CUDA-core conv in fp32 (_video_dgrad).  Gradients are checked against the unmodified reference's autograd on the `mini`
  config (tests/golden/mini_train.pt, tests/test_train_gpu.py).

Reference lines: M: = magvit2_pytorch/magvit2_pytorch.py, A: = attend.py.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, List, Sequence

import torch
import torch.nn.functional as F

from ._lib import ACT_ELU
from .dist import LFQ_DENSE_MAX_D
from .engine import Engine, pack_conv


# --------------------------------------------------------------------------------------------
# torch restatements of the light blocks, channels-last (B, T, H, W, C) -- used for the backward only
# --------------------------------------------------------------------------------------------
def _rmsnorm(x, gamma):
    """RMSNorm (M:275-276): F.normalize over channels * sqrt(C) * gamma."""
    return F.normalize(x, dim=-1) * (x.shape[-1] ** 0.5) * gamma.reshape(-1)


def _token_shift(x):
    """TokenShift (M:250-254): the second chunk of the channels delayed by one frame, zeros at t = 0."""
    a, s = x.chunk(2, dim=-1)
    s = F.pad(s, (0, 0, 0, 0, 0, 0, 1, -1))
    return torch.cat((a, s), dim=-1)


def _squeeze_excite(y, se):
    """SqueezeExcite (M:221-240) on (B,T,H,W,C): per frame, softmax-pooled channel vector -> 2-layer MLP -> sigmoid gate."""
    B, T, H, W, Cc = y.shape
    yf = y.reshape(B * T, H * W, Cc)
    logits = yf @ se.to_k.weight.reshape(Cc) + se.to_k.bias
    attn = logits.float().softmax(dim=-1).to(y.dtype)
    pooled = torch.einsum("fp,fpc->fc", attn, yf)
    hd = se.net[0].weight.shape[0]
    hid = F.leaky_relu(F.linear(pooled, se.net[0].weight.reshape(hd, Cc), se.net[0].bias), 0.1)
    gate = torch.sigmoid(F.linear(hid, se.net[2].weight.reshape(Cc, hd), se.net[2].bias))
    return (yf * gate[:, None, :]).reshape(y.shape)


def dropout_scale(p: float) -> float:
    """fp32(1 / (1 - p)) of the fp32 value of p: the factor the attention kernels apply to the kept weights."""
    return C.c_float(1.0 / (1.0 - C.c_float(p).value)).value


def _softmax_attention(q, k, v, causal, dropout=None):
    """Attend (A:218-241) with the right-aligned causal mask (A:46-47, A:123-129).  `dropout`: (keep mask (b, h, i, j) uint8, p)
    -- the softmax weights are multiplied by keep * fp32(1 / (1 - p)) after the softmax (A:239)."""
    dots = torch.einsum("bhid,bhjd->bhij", q, k) * (q.shape[-1] ** -0.5)
    i, j = dots.shape[-2:]
    if causal and i > 1:
        mask = torch.ones((i, j), dtype=torch.bool, device=q.device).triu(j - i + 1)
        dots = dots.masked_fill(mask, -torch.finfo(dots.dtype).max)
    attn = dots.softmax(dim=-1)
    if dropout is not None:
        keep, p = dropout
        attn = attn * keep.to(attn.dtype) * dropout_scale(p)
    return torch.einsum("bhij,bhjd->bhid", attn, v)


def _attention_block(x, at, axis, dropout=None):
    """Residual(SpaceAttention) / Residual(TokenShift(TimeAttention)) (M:327-388, M:444-464, M:1190, M:1235).  `dropout`: as
    _softmax_attention's, the mask laid out as mv2_attention_dropout_mask writes it."""
    B, T, H, W, Cc = x.shape
    xs = _token_shift(x) if axis == "time" else x
    xn = _rmsnorm(xs, at.norm.gamma)
    tok = xn.permute(0, 2, 3, 1, 4).reshape(B * H * W, T, Cc) if axis == "time" else xn.reshape(B * T, H * W, Cc)
    b, n, _ = tok.shape
    qkv = F.linear(tok, at.to_qkv[0].weight).reshape(b, n, 3, at.heads, -1).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    mem = at.mem_kv.to(x.dtype)
    k = torch.cat((mem[0][None].expand(b, -1, -1, -1), k), dim=-2)
    v = torch.cat((mem[1][None].expand(b, -1, -1, -1), v), dim=-2)
    o = _softmax_attention(q, k, v, causal=(axis == "time"), dropout=dropout).permute(0, 2, 1, 3).reshape(b, n, -1)
    o = F.linear(o, at.to_out[1].weight)
    o = o.reshape(B, H, W, T, Cc).permute(0, 3, 1, 2, 4) if axis == "time" else o.reshape(B, T, H, W, Cc)
    return o + x


def _linear_attention_block(x, la):
    """Residual(LinearSpaceAttention) (M:390-442) with the Taylor-series linear attention of SURVEY Appendix A.3."""
    B, T, H, W, Cc = x.shape
    heads, dh = la.heads, la.dim_head
    tok = _rmsnorm(x, la.norm.gamma).reshape(B * T, H * W, Cc)
    b, n, _ = tok.shape
    q = F.linear(tok, la.attn.to_q[0].weight).reshape(b, n, heads, dh).permute(0, 2, 1, 3) * dh ** -0.5
    kv = F.linear(tok, la.attn.to_kv[0].weight).reshape(b, n, 2, heads, dh).permute(2, 0, 3, 1, 4)
    k, v = kv[0], kv[1]

    def phi(z):
        one = z.new_ones((*z.shape[:-1], 1))
        z2 = (z[..., :, None] * z[..., None, :]) * (0.5 ** 0.5)
        return torch.cat((one, z, z2.reshape(*z.shape[:-1], -1)), dim=-1)

    q, k = phi(q), phi(k)
    kvs = torch.einsum("bhnd,bhne->bhde", k, v)
    num = torch.einsum("bhnd,bhde->bhne", q, kvs)
    den = torch.einsum("bhnd,bhd->bhn", q, k.sum(dim=-2))[..., None]
    o = (num / den.clamp(min=1e-5)).permute(0, 2, 1, 3).reshape(b, n, heads * dh)
    return F.linear(o, la.attn.to_out[0].weight).reshape(x.shape) + x


def _gateloop_block(x, gl):
    """ToTimeSequence(Residual(SimpleGateLoopLayer)) (M:178-191, M:1216-1222): s_t = sigmoid(a_t) s_{t-1} + kv_t, out_t = q_t s_t."""
    q, kv, a = F.linear(_rmsnorm(x, gl.norm.gamma), gl.to_qkva[0].weight).chunk(3, dim=-1)
    a = a.sigmoid()
    s = torch.zeros_like(kv[:, 0])
    outs = []
    for t in range(x.shape[1]):
        s = a[:, t] * s + kv[:, t]
        outs.append(q[:, t] * s)
    return torch.stack(outs, dim=1) + x


def _residual_unit_mod(x, cond_e, mod):
    """ResidualUnitMod (M:946-988) with Conv3DMod (M:718-753): per-clip weights w (cond + 1), demodulated by rsqrt(sum w_b^2),
    one grouped causal conv over the batch; ELU; 1x1x1 conv; ELU; residual.  x (B,T,H,W,C), cond_e (B, dim_cond)."""
    B, T, H, W, Cc = x.shape
    c = F.linear(cond_e.to(x.dtype), mod.to_cond.weight, mod.to_cond.bias)
    w = mod.conv.weights
    o, i, kt, kh, kw = w.shape
    wb = w[None] * (c[:, None, :, None, None, None] + 1.)
    wb = wb * (wb ** 2).sum(dim=(2, 3, 4, 5), keepdim=True).clamp(min=mod.conv.eps).rsqrt()
    xc = x.permute(0, 4, 1, 2, 3)
    xg = F.pad(xc.reshape(1, B * i, T, H, W), (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    y = F.elu(F.conv3d(xg, wb.reshape(B * o, i, kt, kh, kw), groups=B).reshape(B, o, T, H, W))
    y = F.elu(F.conv3d(y, mod.conv_out.weight, mod.conv_out.bias))
    return (y + xc).permute(0, 2, 3, 4, 1)


def _feed_forward_block(x, ff, shift):
    """Residual(FeedForward) / Residual(TokenShift(FeedForward)) (M:466-508, M:1191, M:1236)."""
    xs = _token_shift(x) if shift else x
    xn = _rmsnorm(xs, ff.norm.gamma)
    w1, w2 = ff.net[0].weight, ff.net[2].weight
    hdn = F.linear(xn, w1.reshape(w1.shape[0], -1), ff.net[0].bias)
    a, gate = hdn.chunk(2, dim=-1)
    return F.linear(F.gelu(gate) * a, w2.reshape(w2.shape[0], -1), ff.net[2].bias) + x


def _upsample_space(x, conv):
    """SpatialUpsample2x (M:811-846): 1x1 conv C -> 4 C', SiLU, 'b (c p1 p2) h w -> b c (h p1) (w p2)'."""
    B, T, H, W, _ = x.shape
    w = conv.weight
    o = F.silu(F.linear(x, w.reshape(w.shape[0], -1), conv.bias))
    co = o.shape[-1] // 4
    return o.reshape(B, T, H, W, co, 2, 2).permute(0, 1, 2, 5, 3, 6, 4).reshape(B, T, 2 * H, 2 * W, co)


def _upsample_time(x, conv):
    """TimeUpsample2x (M:848-883): 1x1 conv C -> 2 C', SiLU, 'b (c p) t -> b c (t p)'."""
    B, T, H, W, _ = x.shape
    w = conv.weight
    o = F.silu(F.linear(x, w.reshape(w.shape[0], -1), conv.bias))
    co = o.shape[-1] // 2
    return o.reshape(B, T, H, W, co, 2).permute(0, 1, 5, 2, 3, 4).reshape(B, 2 * T, H, W, co)


def _entropy(p, eps=1e-5):
    return (-p * torch.log(p.clamp(min=eps))).sum(dim=-1)


def _lfq_project(x, qz):
    """LFQ's pre-sign values (SURVEY Appendix A.1 steps 2-4) on (B,T,H,W,C): project_in, soft clamp, [spherical] -> fp32 (N, nc, d)."""
    d, nc = qz.codebook_dim, qz.num_codebooks
    p = F.linear(x, qz.project_in.weight, qz.project_in.bias)
    cv = qz.soft_clamp_input_value
    if cv:
        p = (p / cv).tanh() * cv
    p = p.reshape(-1, nc, d)
    if qz.spherical:
        p = F.normalize(p, dim=-1)
    return p.float()


def _lfq_quantize(x, qz, straight_through):
    """LFQ's quantised output without the auxiliary loss (the first element of encode(quantize=True)): project_out of the
    signs, with the straight-through estimator x + (q - x).detach() in train mode (A.1 step 6); in eval mode the signs are a
    constant of the input, so only project_out gets a gradient."""
    p = _lfq_project(x, qz)
    qd = torch.where(p > 0, torch.ones_like(p), -torch.ones_like(p))
    st = p + (qd - p).detach() if straight_through else qd.detach()
    return F.linear(st.reshape(*x.shape[:-1], -1).to(x.dtype), qz.project_out.weight, qz.project_out.bias)


def _project_out(codes, qz, dtype):
    """indices_to_codes' projection (M:1593): project_out of the code values (B,T,H,W, nc * d) -- the only parameters
    decode_from_code_indices reaches in the quantiser."""
    return F.linear(codes.to(dtype), qz.project_out.weight, qz.project_out.bias)


def _code_values(codes, qz, fsq):
    """Code values (B,T,H,W, nc * d) fp32 of indices (B,T,H,W[,nc]): LFQ's +-1 bits, FSQ's (level - half width) / half width
    (indices_to_codes, A.1 / A.2)."""
    ind = codes.long().reshape(*codes.shape[:4], -1)[..., None]                   # (B,T,H,W,nc,1)
    if fsq:
        lv = torch.tensor(qz.levels, device=codes.device, dtype=torch.long)
        basis = torch.cumprod(torch.cat((lv.new_ones(1), lv[:-1])), dim=0)
        half = lv // 2
        vals = ((ind // basis) % lv - half).float() / half.float()
    else:
        vals = ((ind & qz.mask.to(codes.device).long()) != 0).float() * 2 - 1
    return vals.reshape(*codes.shape[:4], -1)


def _lfq_train(x, qz, avg_global, eng=None, inv_temperature=100.):
    """LFQ training forward (SURVEY Appendix A.1 steps 2-10) on (B,T,H,W,C): -> (straight-through quantised output, aux loss).
    `avg_global` is the cross-rank mean code probability of the forward pass; the local term enters as
    avg_local + (avg_global - avg_local).detach(), which reproduces the gradient of the reference's autograd-aware
    all-reduce (each rank back-propagates d H / d avg_global into its own tokens).  `eng`: the Engine that launches (and
    counts) the bit-factorised entropy kernels of codebooks past 2^LFQ_DENSE_MAX_D codes; None: an engine of the call's own."""
    d, nc = qz.codebook_dim, qz.num_codebooks
    p = _lfq_project(x, qz)
    qd = torch.where(p > 0, torch.ones_like(p), -torch.ones_like(p))
    st = (p + (qd - p).detach()).reshape(*x.shape[:-1], nc * d)
    out = F.linear(st.to(x.dtype), qz.project_out.weight, qz.project_out.bias)
    commit = ((p - qd) ** 2).mean()
    if d > LFQ_DENSE_MAX_D:
        if eng is None:
            eng = Engine(None)
            eng.bind(p, "the LFQ entropy terms")
        ent = _LfqEntropyFact.apply(eng, p.contiguous(), avg_global.reshape(-1).float().contiguous(), inv_temperature,
                                    qz.entropy_loss_weight, qz.diversity_gamma)
        return out, ent + commit * qz.commitment_loss_weight
    mask = qz.mask.to(p.device)
    codebook = ((torch.arange(2 ** d, device=p.device)[:, None] & mask) != 0).float() * 2 - 1
    prob = (2 * inv_temperature * torch.einsum("tcd,kd->tck", p, codebook)).softmax(dim=-1)      # (tokens, nc, K)
    per_sample = _entropy(prob).mean()
    avg_local = prob.mean(dim=0)                                                                  # (nc, K)
    avg = avg_local + (avg_global.reshape(nc, -1) - avg_local).detach()
    aux = (per_sample - qz.diversity_gamma * _entropy(avg).mean()) * qz.entropy_loss_weight + commit * qz.commitment_loss_weight
    return out, aux


class _LfqEntropyFact(torch.autograd.Function):
    """The entropy part of LFQ's aux loss, entropy_weight * (per_sample_entropy - diversity_gamma * batch_entropy), for
    codebooks of 2^13 .. 2^20 codes, where the dense (tokens, nc, 2^d) probabilities of _lfq_train's d <= 12 path would take
    gigabytes.  The code distribution factorises over bits (DESIGN.md), so the value comes from mv2_lfq_entropy_fact_partials
    and mv2_lfq_aux_finalize and the gradient of the pre-sign values from mv2_lfq_entropy_fact_backward, both O(tokens 2^d)
    with no per-token table of size 2^d.  The batch term is taken at the cross-rank mean `avg_global`, whose gradient reaches
    the local tokens as through _lfq_train's avg_local + (avg_global - avg_local).detach()."""

    @staticmethod
    def forward(ctx, eng, p, avg_global, inv_temperature, entropy_weight, diversity_gamma):
        N, nc, d = p.shape
        dev = p.device
        ws = torch.empty(eng.lib.mv2_lfq_entropy_fact_workspace_bytes(N, d, nc), device=dev, dtype=torch.uint8)
        avg_local = torch.empty(nc << d, device=dev, dtype=torch.float32)
        stats = torch.empty(2, device=dev, dtype=torch.float32)
        eng._call("mv2_lfq_entropy_fact_partials", p.data_ptr(), N, d, nc, float(inv_temperature), avg_local.data_ptr(),
                  stats.data_ptr(), ws.data_ptr())
        out4 = torch.empty(4, device=dev, dtype=torch.float32)
        # avg_global is already a mean (n_tokens_global = 1); out4 = (per_sample, batch_entropy, commitment, aux) with the
        # commitment left to autograd (weight 0 here)
        eng._call("mv2_lfq_aux_finalize", avg_global.data_ptr(), stats.data_ptr(), d, nc, N, 1, float(diversity_gamma),
                  float(entropy_weight), 0.0, out4.data_ptr())
        ctx.save_for_backward(p, avg_global)
        ctx.eng = eng
        ctx.coefs = (float(inv_temperature), entropy_weight / (N * nc), entropy_weight * diversity_gamma / (N * nc))
        return out4[3].clone()

    @staticmethod
    def backward(ctx, g):
        eng = ctx.eng
        p, avg_global = ctx.saved_tensors
        N, nc, d = p.shape
        inv_t, coef_sample, coef_batch = ctx.coefs
        ws = torch.empty(eng.lib.mv2_lfq_entropy_fact_workspace_bytes(N, d, nc), device=p.device, dtype=torch.uint8)
        gp = torch.empty_like(p)
        eng._call("mv2_lfq_entropy_fact_backward", p.data_ptr(), avg_global.data_ptr(), N, d, nc, inv_t, coef_sample, coef_batch,
                  gp.data_ptr(), ws.data_ptr())
        return None, gp * g, None, None, None, None


def _fsq_train(x, qz):
    """FSQ forward (SURVEY Appendix A.2) with the round() straight-through estimator."""
    lv = torch.tensor(qz.levels * qz.num_codebooks, dtype=torch.int32, device=x.device)     # the levels repeat per codebook
    z = F.linear(x, qz.project_in.weight, qz.project_in.bias).float()
    half_l = (lv - 1) * (1 + 1e-3) / 2
    offset = torch.where(lv % 2 == 0, 0.5, 0.0)
    bounded = (z + (offset / half_l).atanh()).tanh() * half_l - offset
    quant = bounded + (bounded.round() - bounded).detach()
    return F.linear((quant / (lv // 2)).to(x.dtype), qz.project_out.weight, qz.project_out.bias)


# --------------------------------------------------------------------------------------------
# the tape
# --------------------------------------------------------------------------------------------
def _elu_grad(g, y):
    """d ELU(x) / dx from the OUTPUT y = ELU(x): 1 for x > 0 (y > 0), exp(x) = y + 1 otherwise."""
    return g * torch.where(y > 0, torch.ones_like(y), y + 1)


def transposed_pack(weight, k, dtype):
    """The weight pack of a stride-1 conv's data gradient: weight (Co, Ci, *k) flipped in (t, h, w) and transposed in
    (co, ci), so that the transposed conv is the same implicit GEMM on the engine's conv kernels."""
    kt, kh, kw = k
    wt = weight.detach().reshape(weight.shape[0], -1, kt, kh, kw).flip(2, 3, 4).transpose(0, 1).contiguous()
    return pack_conv(wt, None, dtype)


class TapeRunner:
    """A forward through the engine's kernels that records its backward on a tape, with the tape loop and the gradient
    pieces shared by the generator's runner (TrainRunner), the discriminator's (gan.DiscrRunner) and the VGG's
    (vgg.VggRunner)."""

    def __init__(self, eng):
        self.eng = eng
        self.tape: List[Callable] = []
        self.grads: Dict[torch.nn.Parameter, torch.Tensor] = {}
        self.own_dgrad = True            # data gradient of the stride-1 convs through the engine's own conv kernels
        self.own_dgrad_calls = 0

    def _run_tape(self, g, msg):
        """Runs the tape in reverse from g under no_grad, up to an entry that returns None, then drops it: its closures refer
        to this runner, so the saved activations are freed with the loss graph, not at a later cyclic collection.  `msg`:
        the error of a second backward."""
        if not self.tape:
            raise RuntimeError(msg)
        with torch.no_grad():
            for entry in reversed(self.tape):
                g = entry(g)
                if g is None:
                    break
        self.tape = []
        return g

    # ---- gradient bookkeeping
    def _acc(self, param, g):
        if g is None or not param.requires_grad:
            return
        g = g.reshape(param.shape).to(param.dtype)
        self.grads[param] = g if param not in self.grads else self.grads[param] + g

    def _vjp(self, fn, x, params: Sequence[torch.nn.Parameter], gout, extra=None):
        """Gradient of the block fn at its saved input x: re-evaluates the torch restatement under autograd.  `extra`: further
        leaf tensors (requires_grad) the block reads; their gradients are returned as the second element of a tuple."""
        x_ = x.detach().requires_grad_(True)
        params = [p for p in params if p.requires_grad]
        extra = list(extra or [])
        with torch.enable_grad():
            out = fn(x_)
        outs, gouts = (list(out), list(gout)) if isinstance(out, (tuple, list)) else ([out], [gout])
        gs = torch.autograd.grad(outs, [x_] + params + extra, gouts, allow_unused=True)
        for p, g in zip(params, gs[1:1 + len(params)]):
            self._acc(p, g)
        if extra:
            return gs[0], gs[1 + len(params):]
        return gs[0]

    # ---- conv gradients
    def _dgrad(self, g, weight, k, out_spatial):
        """Data gradient of a stride-1 conv with leading pad (kt - 1, kh // 2, kw // 2) on the engine's conv kernels: the
        transposed conv is the same implicit GEMM with the weights flipped in (t, h, w) and transposed in (co, ci), and no
        leading pad in time (gx[t] = sum_e W'[e] g[t + e]; frames past the clip are the kernels' out-of-bounds zeros).
        g: (B,To,Ho,Wo,Co) channels-last; returns (B,*out_spatial,Ci) channels-last."""
        kt, kh, kw = k
        self.own_dgrad_calls += 1
        return self.eng.conv(g.contiguous(), transposed_pack(weight, k, self.eng.dtype), pad=(0, kh // 2, kw // 2),
                             out_spatial=tuple(out_spatial))

    def _wgrad(self, g, x_cf, weight, bias, k, stride, pad, need_gx=False):
        """aten.convolution_backward (cuDNN) of y = conv(x_cf; weight, stride, symmetric pad): accumulates the weight / bias
        gradients and returns the data gradient (B,C,T,H,W) if need_gx.  g: (B,To,Ho,Wo,Co) channels-last."""
        w_grad, b_grad = weight.requires_grad, bias is not None and bias.requires_grad
        if not (need_gx or w_grad or b_grad):
            return None
        w5 = weight.reshape(weight.shape[0], -1, *k)
        gx, gw, gb = torch.ops.aten.convolution_backward(
            g.permute(0, 4, 1, 2, 3), x_cf, w5, [w5.shape[0]] if bias is not None else None, list(stride), list(pad), [1, 1, 1],
            False, [0, 0, 0], 1, [need_gx, w_grad, b_grad])
        self._acc(weight, gw)
        if bias is not None:
            self._acc(bias, gb)
        return gx

    def _conv_bwd(self, g, x, weight, bias, k, stride=(1, 1, 1), pad=None, need_gx=True, x_is_cf=False):
        """Backward of a conv the engine ran as  y = conv(x; leading pad (pt, ph, pw), stride).
        g: (B,To,Ho,Wo,Co) channels-last grad of the pre-activation output; x: the saved channels-last input (or, x_is_cf,
        a (B,C,T,H,W) tensor).  Returns grad wrt x (channels-last) or None.
          * data gradient of the stride-1 causal convs (every ResidualUnit conv, conv_out): _dgrad, on our conv kernels;
          * weight / bias gradients, and the data gradient of the strided down-samplers: _wgrad (cuDNN).  The time axis is
            padded at the FRONT only (causal, M:913-928): those zero frames are materialised; H / W use the symmetric padding
            natively."""
        kt, kh, kw = k
        causal_default = pad is None
        if pad is None:
            pad = (kt - 1, kh // 2, kw // 2)
        pt, ph, pw = pad
        own_dgrad = need_gx and self.own_dgrad and causal_default and tuple(stride) == (1, 1, 1) and not x_is_cf
        gx = self._dgrad(g, weight, k, x.shape[1:4]) if own_dgrad else None
        if x_is_cf:
            x_cf = F.pad(x, (0, 0, 0, 0, pt, 0)) if pt > 0 else x
        else:       # pad the (contiguous) channels-last tensor along T, then view it as (B,C,T,H,W) in channels_last_3d strides
            x_cf = (F.pad(x, (0, 0, 0, 0, 0, 0, pt, 0)) if pt > 0 else x).permute(0, 4, 1, 2, 3)
        gxl = self._wgrad(g, x_cf, weight, bias, k, stride, (0, ph, pw), need_gx=need_gx and not own_dgrad)
        if not need_gx or own_dgrad:
            return gx
        return gxl[:, :, pt:].permute(0, 2, 3, 4, 1).contiguous()


class TrainRunner(TapeRunner):
    """One training-mode forward of the tokenizer through the engine's kernels, recording what the backward needs."""

    def __init__(self, model):
        super().__init__(model.engine)
        self.m = model
        self.g_cond: Dict[str, torch.Tensor] = {}      # gradient wrt the cond stems' outputs, summed over the cond_residual stages
        self.codes = None
        self.breakdown = None
        self._bwd_conv_out = None

    def _conv_bwd_padmode(self, g, x, weight, bias, k, pad_mode, need_gx=True):
        """Backward of Engine.causal_conv_padded (CausalConv3d with pad_mode reflect / replicate / circular, M:925-927): the padding
        is re-applied with F.pad under autograd, the conv backward runs without implicit padding on the padded tensor, and the
        gradient is folded back through the padding.  Falls back to the zero-padded case like the forward (time_pad >= T)."""
        kt, kh, kw = k
        if pad_mode == "constant" or kt - 1 >= x.shape[1]:
            return self._conv_bwd(g, x, weight, bias, k, need_gx=need_gx)
        x_ = x.detach().permute(0, 4, 1, 2, 3).requires_grad_(need_gx)
        with torch.enable_grad():
            xp = F.pad(x_, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0), mode=pad_mode)
        gxp = self._wgrad(g, xp.detach(), weight, bias, k, (1, 1, 1), (0, 0, 0), need_gx=need_gx)
        if not need_gx:
            return None
        gx, = torch.autograd.grad(xp, x_, gxp)
        return gx.permute(0, 2, 3, 4, 1).contiguous()

    # ---- forward pieces (engine kernels) that record their backward
    def _residual_unit(self, x, p, ru):
        """ResidualUnit (M:930-944) unfused: both conv outputs are kept for the backward."""
        eng = self.eng
        seq = ru.fn
        c3m, c1m, se = seq[0].conv, seq[2], seq[4]
        h = eng.conv(x, p["conv3"], act=ACT_ELU)
        y = eng.conv(h, p["conv1"], act=ACT_ELU)
        out = eng.squeeze_excite_residual(y, x, p)
        k3 = tuple(c3m.weight.shape[2:])

        def bwd(g):
            gy = self._vjp(lambda t: _squeeze_excite(t, se), y, list(se.parameters()), g)
            gh = self._conv_bwd(_elu_grad(gy, y), h, c1m.weight, c1m.bias, (1, 1, 1))
            gx = self._conv_bwd(_elu_grad(gh, h), x, c3m.weight, c3m.bias, k3)
            return g + gx

        self.tape.append(bwd)
        return out

    def _attn_keep(self, x, at, axis, drop):
        """(keep mask, p) of the attention call `drop` (its (seed, call, p)) on the block input x, regenerated by
        mv2_attention_dropout_mask when the backward needs it; None without dropout.  The uint8 mask lives only as long as
        the block's backward."""
        if drop is None:
            return None
        B, T, H, W, _ = x.shape
        n_seq, L = (B * H * W, T) if axis == "time" else (B * T, H * W)
        return self.eng.attention_dropout_mask(n_seq, at.heads, L, int(at.mem_kv.shape[2]), drop), drop.p

    def _block(self, x, run, fn, params):
        """A light block: forward by the engine (`run`), backward by the torch restatement `fn` on the saved input."""
        out = run(x)
        self.tape.append(lambda g: self._vjp(fn, x, params, g))
        return out

    def _stage(self, x, st, key, mod, decoder, cond_e=None):
        eng = self.eng
        P = eng._packs
        B, T, H, W, Cc = x.shape
        if st.kind == "cond_residual":
            side = "dec" if decoder else "enc"
            xin = x
            out = eng._stage(x, st, key, decoder=decoder, cond_e=cond_e)

            def bwd(g):
                ce = cond_e.detach().requires_grad_(True)
                gx, (gc,) = self._vjp(lambda t: _residual_unit_mod(t, ce, mod), xin, list(mod.parameters()), g, extra=[ce])
                if gc is not None:
                    self.g_cond[side] = gc if side not in self.g_cond else self.g_cond[side] + gc
                return gx

            self.tape.append(bwd)
            return out
        if st.kind == "residual":
            units = list(mod) if st.nested else [mod]
            for j, ru in enumerate(units):
                x = self._residual_unit(x, P[f"{key}.{j}"], ru)
            return x
        if st.kind in ("compress_space", "compress_time") and not decoder:
            conv = mod.conv
            if st.kind == "compress_space":     # SpatialDownsample2x (M:770-780): Conv2d k3 s2 p1 per frame
                k, stride, pad = (1, 3, 3), (1, 2, 2), (0, 1, 1)
            else:                               # TimeDownsample2x (M:796-807): F.pad (2, 0) + Conv1d k3 s2 per pixel
                k, stride, pad = (3, 1, 1), (2, 1, 1), (2, 0, 0)
            xin = x
            out = eng._stage(x, st, key, decoder=False)
            self.tape.append(lambda g: self._conv_bwd(g, xin, conv.weight, conv.bias, k, stride, pad))
            return out
        run = lambda t: eng._stage(t, st, key, decoder=decoder)       # noqa: E731
        if st.kind == "compress_space":
            conv = mod.net[0]
            return self._block(x, run, lambda t: _upsample_space(t, conv), list(conv.parameters()))
        if st.kind == "compress_time":
            conv = mod.net[0]
            return self._block(x, run, lambda t: _upsample_time(t, conv), list(conv.parameters()))
        if st.kind == "gateloop_time":
            gl = mod.fn.fn
            return self._block(x, run, lambda t: _gateloop_block(t, gl), list(gl.parameters()))
        if st.kind in ("attend_space", "attend_time", "linear_attend_space"):
            time_axis = st.kind == "attend_time"
            at = mod[0].fn.fn if time_axis else mod[0].fn
            ff = mod[1].fn.fn if time_axis else mod[1].fn
            if st.kind == "linear_attend_space":
                x = self._block(x, lambda t: eng.linear_attention(t, P[key + ".attn"]), lambda t: _linear_attention_block(t, at),
                                list(at.parameters()))
            else:
                axis = "time" if time_axis else "space"
                drop = None if eng.dropout is None else eng.dropout.take()
                x = self._block(x, lambda t: eng.attention(t, P[key + ".attn"], axis, *(() if drop is None else (drop,))),
                                lambda t: _attention_block(t, at, axis, self._attn_keep(t, at, axis, drop)), list(at.parameters()))
            return self._block(x, lambda t: eng.feed_forward(t, P[key + ".ff"], token_shift=time_axis),
                               lambda t: _feed_forward_block(t, ff, time_axis), list(ff.parameters()))
        raise NotImplementedError(f"no training path for layer type {st.kind!r}")

    # ---- the three pieces of a forward (encoder, quantiser, decoder); each records its backward on the tape.  The training
    #      forward chains all three, the differentiable encode / decode entry points (run_encode, run_decode, run_decode_codes)
    #      one or two of them
    def encoder_piece(self, video, first_frame=True, cond=None, need_gvideo=False):
        """conv_in + the encoder stages (M:1523-1565): video (B,C,T,H,W) -> encoder output, channels-last.  need_gvideo: the
        backward also returns the video's gradient (B,C,T,H,W) (_conv_in_bwd)."""
        m, eng = self.m, self.eng
        self.cond = cond
        ce = eng.cond_stem(cond, "enc") if m.has_cond else None            # M:1544-1548 (Linear + SiLU stem)
        x = eng.conv_in(video, first_frame)
        self.tape.append(self._conv_in_bwd(video, first_frame, need_gvideo))
        for i, st in enumerate(m.stages):
            x = self._stage(x, st, f"enc{i}", m.encoder_layers[i], decoder=False, cond_e=ce)
        return x

    def _conv_in_bwd(self, vid, first_frame, need_gvideo):
        """conv_in's tape entry: weight / bias gradients of conv_in [and conv_in_first_frame], and with need_gvideo the gradient
        wrt the video (B,C,T,H,W), without the time_padding frames the reference prepends as constants (M:1534-1537).  The
        video's data gradient runs on the engine's conv kernels (_video_dgrad) except in the non-constant pad modes, where it
        is folded back through F.pad like the other padded convs (_conv_bwd_padmode)."""
        m, eng = self.m, self.eng
        t_pad = m.time_padding if first_frame else 0
        cin = m.conv_in.conv
        kin = tuple(cin.weight.shape[2:])
        sff = bool(m.separate_first_frame_encoding and first_frame)
        mode = m.conv_in.pad_mode

        def padded(frames):          # the forward pads with pad_mode (Engine.causal_conv_padded), not with zeros
            return need_gvideo and mode != "constant" and kin[0] - 1 < frames

        def bwd(g):
            # the causal conv_in's input in the pad modes: channels-last, from the same layout kernel as in the forward
            v = (vid.float() / 255. if vid.dtype == torch.uint8 else vid).to(eng.dtype)
            if sff:
                ff = m.conv_in_first_frame
                kff = (1,) + tuple(ff.weight.shape[2:])
                gv = torch.zeros(v.shape, device=v.device, dtype=eng.dtype) if need_gvideo else None
                g0 = g[:, t_pad:t_pad + 1].contiguous()
                self._conv_bwd(g0, v[:, :, 0:1], ff.weight, ff.bias, kff, pad=(0, kff[1] // 2, kff[2] // 2), need_gx=False, x_is_cf=True)
                if need_gvideo:
                    gv[:, :, 0:1] = self._video_dgrad(g0, ff.weight, kff, 0)
                if v.shape[2] > 1:
                    g1 = g[:, t_pad + 1:].contiguous()
                    gx = self._conv_bwd_padmode(g1, eng.to_channels_last(vid[:, :, 1:]), cin.weight, cin.bias, kin, mode,
                                                need_gx=padded(v.shape[2] - 1))
                    if need_gvideo:
                        gv[:, :, 1:] = gx.permute(0, 4, 1, 2, 3) if gx is not None else self._video_dgrad(g1, cin.weight, kin, 0)
                return gv
            if mode != "constant":
                gx = self._conv_bwd_padmode(g, eng.to_channels_last(vid, t_pad), cin.weight, cin.bias, kin, mode,
                                            need_gx=padded(v.shape[2] + t_pad))
            else:
                gx = None
                self._conv_bwd(g, v, cin.weight, cin.bias, kin, pad=(t_pad + kin[0] - 1, kin[1] // 2, kin[2] // 2),
                               need_gx=False, x_is_cf=True)
            if not need_gvideo:
                return None
            return gx[:, t_pad:].permute(0, 4, 1, 2, 3) if gx is not None else self._video_dgrad(g, cin.weight, kin, t_pad)

        return bwd

    def _video_dgrad(self, g, weight, k, t_crop):
        """Data gradient of conv_in (or its first-frame conv) wrt the video on the engine's conv kernels, like _dgrad: the same
        implicit GEMM with flipped / transposed weights (K = taps x init_dim, N = channels), without its first t_crop frames
        (the time_padding).  g: (B,Ti,H,W,init_dim) channels-last -> (B,channels,Ti - t_crop,H,W).  In bf16 the slab kernel's
        narrow N tile writes torch's layout directly (Engine.conv_cf_supported); otherwise the conv's channels-last output is
        transposed."""
        return self.video_dgrad_packed(g, transposed_pack(weight, k, self.eng.dtype), t_crop)

    def video_dgrad_packed(self, g, pk, t_crop):
        """_video_dgrad with the transposed weight pack given (transposed_pack)."""
        eng = self.eng
        _, kh, kw = pk.k
        B, Ti, H, W, _ = g.shape
        self.own_dgrad_calls += 1
        g = g.contiguous()
        pad_cf, out_cf = (-t_crop, kh // 2, kw // 2), (Ti - t_crop, H, W)
        if eng.conv_cf_supported(g, pk, pad_cf, out_cf):
            return eng.conv(g, pk, pad=pad_cf, out_spatial=out_cf, out_cf=True)
        return eng.to_channels_first(eng.conv(g, pk, pad=(0, kh // 2, kw // 2), out_spatial=(Ti, H, W)), t_crop=t_crop)

    def quantizer_piece(self, x, mode, group=None):
        """The quantiser on the encoder output x (channels-last); the codes are left in .codes.
          * mode "loss" (the training forward, M:1705): -> (quantised, aux loss 0-d fp32).  LFQ with its straight-through
            estimator and auxiliary loss (breakdown in .breakdown, batch entropy over `group`), FSQ with round_ste;
          * mode "quantize" (encode(quantize=True), M:1567-1576): -> quantised.  LFQ is straight-through in train mode only
            (in eval the quantised value is a constant of the input), FSQ's round_ste in both modes.  No auxiliary loss."""
        from .dist import LfqBatchEntropy
        m, eng = self.m, self.eng
        qz = m.quantizers
        params = list(qz.parameters())
        if mode == "quantize":
            q, self.codes, _ = eng.quantize_cl(x)
            if m.use_fsq or m.training:
                fn = (lambda t: _fsq_train(t, qz)) if m.use_fsq else (lambda t: _lfq_quantize(t, qz, True))
                self.tape.append(lambda g: self._vjp(fn, x, params, g))
                return q

            def bwd_eval_lfq(g):      # the signs are a constant of x: project_out's gradient only, and nothing reaches x
                if any(p.requires_grad for p in qz.project_out.parameters()):
                    self._vjp(lambda t: _lfq_quantize(t, qz, False), x, params, g)
                return None

            self.tape.append(bwd_eval_lfq)
            return q
        if m.use_fsq:
            q, self.codes, _ = eng.quantize_cl(x)
            aux = torch.zeros((), device=eng.device, dtype=torch.float32)
            self.tape.append(lambda g: self._vjp(lambda t: _fsq_train(t, qz), x, params, g))
            return q, aux
        q, self.codes, pre = eng.quantize_cl(x, want_quantized=True, want_aux=True)
        be = LfqBatchEntropy(eng, num_codebooks=qz.num_codebooks)
        be.start(pre, group)
        avg_sum = be.avg_prob_sum
        ps, bent, commit, aux = be.finish(qz.diversity_gamma, qz.entropy_loss_weight, qz.commitment_loss_weight, group)
        world = torch.distributed.get_world_size(group) if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 1
        avg_global = avg_sum / world
        self.breakdown = (ps, bent, commit)
        # the auxiliary loss's gradient (self._g_aux) enters here, set by backward
        self.tape.append(lambda g: self._vjp(lambda t: _lfq_train(t, qz, avg_global, eng), x, params, (g, self._g_aux)))
        return q, aux

    def codes_piece(self, codes):
        """indices_to_codes (M:1593) on the engine: codes -> quantised channels-last, recording project_out's backward (a
        torch restatement on the code values; the integer codes themselves have no gradient)."""
        m, eng = self.m, self.eng
        qz = m.quantizers
        q = eng.codes_to_quantized_cl(codes)
        vals = _code_values(codes, qz, m.use_fsq)

        def bwd(g):
            self._vjp(lambda t: _project_out(t, qz, eng.dtype), vals, list(qz.project_out.parameters()), g)
            return None

        self.tape.append(bwd)
        return q

    def decoder_piece(self, q, first_frame=True, cond=None):
        """The decoder stages + conv_out (M:1598-1649): quantised channels-last (B,T',H',W',C) -> reconstruction (B,C,T,H,W)."""
        m, eng = self.m, self.eng
        self.cond = cond
        ce = eng.cond_stem(cond, "dec") if m.has_cond else None            # M:1612-1616
        t_pad = m.time_padding if first_frame else 0
        cout = m.conv_out.conv
        sff = bool(m.separate_first_frame_encoding and first_frame)
        mode_out = m.conv_out.pad_mode
        x = q
        for j, st in enumerate(reversed(m.stages)):
            x = self._stage(x, st, f"dec{j}", m.decoder_layers[j], decoder=True, cond_e=ce)
        xo = x
        kout = tuple(cout.weight.shape[2:])
        recon = eng.conv_out(xo, first_frame)

        def bwd_conv_out(g_recon, need_gx=True):    # (B,C,T,H,W) -> channels-last with zero gradient on the cropped time_padding frames
            # need_gx=False: conv_out's weight / bias gradients only (last_layer_weight_grad), the first frame's conv is skipped
            g = g_recon.permute(0, 2, 3, 4, 1)
            if sff:
                off = m.conv_out_first_frame
                kff = (1,) + tuple(off.weight.shape[2:])
                gx = torch.zeros_like(xo) if need_gx else None
                if need_gx:
                    gx[:, t_pad:t_pad + 1] = self._conv_bwd(g[:, 0:1].contiguous(), xo[:, t_pad:t_pad + 1].contiguous(), off.weight, off.bias,
                                                            kff, pad=(0, kff[1] // 2, kff[2] // 2))
                if xo.shape[1] - t_pad > 1:
                    g1 = self._conv_bwd_padmode(g[:, 1:].contiguous(), xo[:, t_pad + 1:].contiguous(), cout.weight, cout.bias, kout, mode_out,
                                                need_gx=need_gx)
                    if need_gx:
                        gx[:, t_pad + 1:] = g1
                return gx
            if t_pad:
                g = F.pad(g, (0, 0, 0, 0, 0, 0, t_pad, 0))
            return self._conv_bwd_padmode(g.contiguous(), xo, cout.weight, cout.bias, kout, mode_out, need_gx=need_gx)

        self.tape.append(bwd_conv_out)
        self._bwd_conv_out = bwd_conv_out
        return recon

    def forward(self, video, first_frame=True, group=None, cond=None):
        """The training forward: -> (recon (B,C,T,H,W), aux_loss 0-d fp32); codes / the LFQ breakdown are left in .codes /
        .breakdown."""
        x = self.encoder_piece(video, first_frame, cond)
        q, aux = self.quantizer_piece(x, "loss", group)
        return self.decoder_piece(q, first_frame, cond), aux

    # ---- the differentiable entry points of VideoTokenizer (one piece chain each); the first tape entry returns the
    #      gradient wrt the call's input in the caller's layout
    def run_encode(self, video, cond, first_frame, quantize, need_gvideo):
        """encode (M:1523-1576): video -> (B,C,T',H',W') encoder output or, quantize, the quantised value."""
        x = self.encoder_piece(video, first_frame, cond, need_gvideo)
        if quantize:
            x = self.quantizer_piece(x, "quantize")
        dt = self.eng.dtype
        self.tape.append(lambda g: g.permute(0, 2, 3, 4, 1).to(dt).contiguous())     # from the (B,C,T',H',W') output
        return self.eng.to_channels_first(x)

    def run_decode(self, quantized, cond, first_frame):
        """decode (M:1598-1649): quantized (B,C,T',H',W') -> reconstruction."""
        self.tape.append(lambda g: g.permute(0, 4, 1, 2, 3))                          # to the (B,C,T',H',W') input
        return self.decoder_piece(self.eng.to_channels_last(quantized), first_frame, cond)

    def run_decode_codes(self, codes, cond, first_frame):
        """decode_from_code_indices (M:1579-1595): codes (B,T',H',W'[,nc]) -> reconstruction."""
        return self.decoder_piece(self.codes_piece(codes), first_frame, cond)

    def last_layer_weight_grad(self, g_recon):
        """The gradient of ``conv_out.conv.weight`` for a reconstruction gradient g_recon (B,C,T,H,W): the adaptive adversarial
        weight's gradient norms at the last decoder layer (M:1812-1841).  Runs conv_out's weight-gradient piece of the tape on the
        saved decoder output; the tape stays intact for the backward and ``self.grads`` is left untouched."""
        if self._bwd_conv_out is None:
            raise RuntimeError("the tokenizer's backward ran already: its saved activations are released")
        w = self.m.conv_out.conv.weight
        grads, self.grads = self.grads, {}
        try:
            with torch.no_grad():
                self._bwd_conv_out(g_recon.to(self.eng.dtype), need_gx=False)
            gw = self.grads.get(w)
        finally:
            self.grads = grads
        return torch.zeros_like(w) if gw is None else gw

    def backward(self, g_out, g_aux=None):
        """Runs the tape in reverse from the gradient of the last piece's output (g_out; g_aux: the auxiliary loss's, training
        forward only) -> (gradient wrt the first piece's input | None, gradient wrt cond | None, {Parameter: grad}).  The
        eval-mode LFQ quantiser's entry returns None: nothing before it is reached."""
        self._g_aux = (g_aux if g_aux is not None else torch.zeros((), device=self.eng.device)).float()
        g = self._run_tape(g_out.to(self.eng.dtype),
                           "the tokenizer's backward ran already: the saved activations are released after one backward pass "
                           "(call the forward again; retain_graph is not supported by this path)")
        self._bwd_conv_out = None          # conv_out's piece of the tape, released with it
        g_cond = None
        for side, stem in (("enc", self.m.encoder_cond_in), ("dec", self.m.decoder_cond_in)):
            if side in self.g_cond:       # cond stems (M:1344-1352): Linear + SiLU of the raw cond vector
                lin = stem[0]
                gc = self._vjp(lambda t, lin=lin: F.silu(F.linear(t, lin.weight.float(), lin.bias.float())), self.cond.float(),
                               list(lin.parameters()), self.g_cond[side].float())
                g_cond = gc if g_cond is None else g_cond + gc
        return g, g_cond, self.grads


class _TapeFn(torch.autograd.Function):
    """(x, cond, *parameters) -> the outputs of `run(x, cond)`, a chain of a runner's pieces on the engine's kernels;
    backward by the runner's tape.  x is the call's input (video, quantised latents or integer codes); the outputs are a
    tensor or, for the training forward, (recon, aux_loss).  Gradients go to x and cond when they are floating, and to
    every parameter handed over."""

    @staticmethod
    def forward(ctx, runner, run, x, cond, *params):
        out = run(x, cond)
        ctx.runner, ctx.params = runner, params
        ctx.in_dtypes = tuple(t.dtype if t is not None and t.is_floating_point() else None for t in (x, cond))
        return out

    @staticmethod
    def backward(ctx, g_out, *g_more):
        gx, gc, grads = ctx.runner.backward(g_out, g_more[0] if g_more else None)
        g_in = tuple(None if (g is None or dt is None) else g.to(dt) for g, dt in zip((gx, gc), ctx.in_dtypes))
        # every parameter handed to the Function gets a gradient tensor (zeros if this call did not touch it, e.g. conv_in of a
        # one-frame clip with separate_first_frame_encoding): DistributedDataParallel waits for the hook of every parameter it can
        # reach from the outputs
        return (None, None) + g_in + tuple(grads[p] if p in grads else torch.zeros_like(p) for p in ctx.params)


def live_parameters(model, first_frame=True):
    """The parameters a forward can reach.  Left out, exactly like in the reference's graph (so DistributedDataParallel must be
    built with find_unused_parameters=True there as here): the final LayerNorm of the encoder, which is constructed but never
    executed (M:1322-1326, M:1565), and the first-frame convs unless separate_first_frame_encoding applies to this call."""
    dead = {id(p) for p in model.encoder_layers[len(model.stages)].parameters()}
    if not (model.separate_first_frame_encoding and first_frame):
        dead |= {id(p) for mod in (model.conv_in_first_frame, model.conv_out_first_frame) for p in mod.parameters()}
    return [p for p in model.parameters() if p.requires_grad and id(p) not in dead]


def reached_parameters(model, entry, first_frame=True, frames=None, quantize=False):
    """The parameters (requires_grad) a differentiable call reaches: those the reference's graph gives a gradient.
      * "decode": the decoder stages, conv_out, conv_out_first_frame (separate_first_frame_encoding with a first frame),
        decoder_cond_in;  "decode_codes": those and quantizers.project_out (indices_to_codes, M:1593);
      * "encode": conv_in, conv_in_first_frame (as above), the encoder stages (not the final LayerNorm, see live_parameters),
        encoder_cond_in; quantize adds the quantiser's projections -- in eval mode only LFQ's project_out, as the signs are a
        constant of the input there.
    frames: the clip's frames (encode) or the decoder's output frames (decode): with separate_first_frame_encoding and a
    first frame, the causal conv_in / conv_out only run on frames after the first."""
    m = model
    sff = bool(m.separate_first_frame_encoding and first_frame)
    mods = []
    if entry == "encode":
        qz = m.quantizers
        if quantize and not m.use_fsq and not m.training:
            return [p for p in qz.project_out.parameters() if p.requires_grad]
        if not (sff and frames == 1):
            mods.append(m.conv_in)
        if sff:
            mods.append(m.conv_in_first_frame)
        mods += [m.encoder_layers[i] for i in range(len(m.stages))] + [m.encoder_cond_in]
        if quantize:
            mods += [qz.project_in, qz.project_out]
    else:
        if entry == "decode_codes":
            mods.append(m.quantizers.project_out)
        mods += [m.decoder_layers, m.decoder_cond_in]
        if not (sff and frames == 1):
            mods.append(m.conv_out)
        if sff:
            mods.append(m.conv_out_first_frame)
    ids = {id(p) for mod in mods for p in mod.parameters()}
    return [p for p in m.parameters() if p.requires_grad and id(p) in ids]


def train_forward(model, video, first_frame=True, cond=None, runner=None):
    """-> (recon with grad_fn, aux_loss with grad_fn, codes, lfq breakdown | None).  `runner`: a fresh TrainRunner of the model
    to run on (the caller keeps it for last_layer_weight_grad)."""
    runner = runner or TrainRunner(model)
    params = live_parameters(model, first_frame)
    recon, aux = _TapeFn.apply(runner, lambda v, c: runner.forward(v, first_frame, cond=c), video, cond, *params)
    return recon, aux, runner.codes, runner.breakdown
