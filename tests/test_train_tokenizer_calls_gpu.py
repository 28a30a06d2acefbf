"""Every kernel call the tokenizer's own engine makes in the README training step's generator step, at the trainer's own
shapes, checked one call at a time against float64: the half of the step tests/test_train_calls_gpu.py (discriminator and
VGG) leaves out.

The workload is that file's: _model() (README_TRAIN_KW, a full VGG16, synth_data weights, bf16, train() with the VGG in
eval()), 4 clips of 3 x 17 x 128 x 128, one warm-up step, then one generator step (return_loss=True, then .backward()).
The training forward differs from the benchmark's eval forward (tests/test_bench_calls_gpu.py): TrainRunner runs every
ResidualUnit unfused (conv3 with ELU, conv1 with ELU, squeeze_excite_residual), the quantiser returns its pre-sign values
and the LFQ batch-entropy terms run on them, and the backward runs the engine's data gradients and cuDNN's weight gradients.
Only model.engine and the runners' methods on it are wrapped; the discriminator's and the VGG's calls pass through.

Part 1, real data.  Each call is checked when it returns (synchronise, float64 reference from the call's own operands one
clip at a time, check, free); every output starts NaN-filled between sentinels (_Guard).  The references and bounds are
the kernel tests', reused through the benchmark test's recorder:
  * Engine.conv (the kw-packed conv_in, the unfused ResidualUnit convs, the down-space and time-strided down-samplers, the
    depth-to-space / depth-to-time up-samplers, the q / kv / qkv / out projections, the GEGLU fc1 and fc2, the
    channels-first conv_out): forward64 / geglu64 (tests/test_conv_forward_gpu.py);
  * squeeze_excite_residual (mv2_se_pool / mv2_se_gate with a softmax pool over 16384 positions of 80 frames at 128^2,
    mv2_gate_residual): the gates within GATE_TOL of _se_gates64 of the kernel's own y, then the gated residual;
  * rmsnorm: _rms_ref;  quantize_cl(want_aux=True): the benchmark test's check, with aux (the pre-sign values) against
    float64;
  * LfqBatchEntropy.start / finish (mv2_lfq_entropy_partials, mv2_lfq_aux_finalize): the float64 dense enumeration of
    tests/test_simt_ops_gpu.py (_lfq_entropy64) on the kernel's own pre-sign input, with that test's relative bounds.
    Those bounds carry the block-count term 8 nblk u, which is the allowance for the fp32 atomic adds derived here: stats[0]
    is the sum of 8 nblk warp partials (one atomicAdd per warp, 8 warps per block), stats[1] of nblk block partials, and
    each avg_prob entry of nblk block partials; all are non-negative, and n non-negative terms summed in any order, each
    addition rounding to nearest, are within (n - 1) u of their sum (Higham 3.1).  Here N = 4 x 5 x 16 x 16 = 5120 tokens,
    nblk = 160 blocks of LE_TOK = 32.  That test's operands lie on a grid where the code logits 2 tau <p, c> are exact;
    the kernel's own pre-sign values are not.  The logit s = fl(sum_i +-p_i) (d - 1 additions) times 2 tau, and the
    kernel's s - max, are within e_t = 1.001 (d + 2) u 2 tau sum_i |p_t,i| of their exact values for every code of token t
    (every partial sum and s - max is at most 2 tau sum |p| in size; 1.001 covers the second-order terms), so each of the
    token's probabilities is within a factor exp(+-2 e_t) of the exact one: |dp| <= D_t p, D_t = expm1(2 e_t).  Its
    avg_prob terms then move by D_t prob_t,k, its entropy by D_t (sum_k x |log x| + 1 + 2 e_t) (|d(-x log x) / dx| <=
    |log x| + 1, and log x moves by at most 2 e_t).  expf / logf (no fast math) stay in the base allowance.  start()
    divides avg_prob by N (one more rounding, u).  mv2_lfq_aux_finalize's four outputs are
    checked against float64 within that test's 1e-4 relative bound;
  * TapeRunner._dgrad (two per ResidualUnit, conv_out's on the CUDA cores): _dgrad64 (tests/test_conv_grad_gpu.py) with
    the gamma(Co taps, C_OF) allowance, one clip at a time against that clip's reference alone, so a read of the next
    clip's frames fails.
The attention kernels are left out, as in the two other call tests: test_attention_gpu.test_readme_forward_attention_calls
checks every mv2_attention / mv2_linear_attention call of a README forward, at this step's sequence lengths (256 tokens
in space, 5 frames in time, 1024 for the linear attention) on one clip instead of four.  The torch restatements the
backward differentiates with _vjp are not kernels; the *_train goldens cover them.

Part 2, exact replay.  Every distinct wgmma call (forward conv or data gradient) runs again on REPLAY_GRID operands with
the same entry point, packer and arguments; at every depth here (up to 512 x 27 = 13824, within the 27 x 1024 up to which
tests/test_bench_calls_cpu.py shows the grid exact) the fp32 accumulation is exact, so the allowance is the epilogue's
alone.  On every slab conv and data gradient whose tiles map one to one onto output channels (not the GEGLU fc1, the
shuffled up-samplers, the kw-packed conv_in) the bound must reject one ring stage missing at the schedule's last tile and
that tile's accumulators not reset (every slab call here plans more tiles than CTAs, so the last tile's CTA ran an earlier
one; tests/test_train_calls_cpu.py).  The down-space flavour has no tile query and is replayed without defects; no
tokenizer call runs on the tap-wise kernel.

Part 3, weight and strided data gradients.  TapeRunner._conv_bwd (and TrainRunner._conv_bwd_padmode, which delegates to
it for the constant pad of conv_out) is wrapped: every conv's weight and bias gradient, the down-samplers' data gradients
and conv_in's channels-first branch go through it.  Each distinct call (shapes, the saved input's strides, k, stride,
pad, need_gx, x_is_cf) is replayed through the same method, its weight gradients captured in an empty runner.grads as
last_layer_weight_grad does, on operands in {-1, 0, 1} laid out with the recorded strides, against float64 autograd of the
forward the engine ran (_conv64_grads).  The deepest sum is 4 x 20 x 128^2 = 1310720 < 2^24 products in {-1, 0, 1}: every
partial sum is an integer below 2^24 and exact in fp32 in any order, so the only allowance is half an ulp of bf16.  This
rests on cuDNN's bf16 convolution backward accumulating in fp32, which the check asserts.  Real-data weight gradients are
not checked against a bound: at depth 1.3M, gamma(K, 2) is 0.16 of the absolute-value sum, which no layout error exceeds.

Negative controls, each rejected: dgrad time taps not flipped; clip i+1's first two frames bled into clip i's last frames;
the SE gates of the last frame taken from the first; one 32-token block left out of avg_prob and the entropy sums;
(replay) the weight gradient with the time pad at the back, or with g one frame late; (replay) the time down-sampler's data
gradient cropped one frame early.

Structure: the calls per kind equal tokenizer_counts of tests/test_train_calls_cpu.py; every call ran the kernel of
tokenizer_table() (conv_out's data gradient is the only CUDA-core conv); from mv2_tc_slab_plan with the device's SM count
the 128^2 unfused ResidualUnit convs and their data gradients ran more than two tiles per CTA."""
import math
import time

import pytest
import torch
import torch.nn.functional as F

import synth_data
from tests.test_bench_calls_gpu import _Recorder as _BenchRecorder
from tests.test_bench_calls_gpu import _defect_deltas, _grid, _lib_plan, _replay_key
from tests.test_conv_forward_gpu import _ran, forward64
from tests.test_conv_grad_gpu import C_OF, _conv64_grads, _dgrad64, _gamma
from tests.test_simt_ops_gpu import U, _check, _lfq_entropy64, _rejects
from tests.test_train_calls_cpu import CLIPS, FRAMES, TOK_SIMT_BY_DESIGN, tokenizer_counts, tokenizer_table
from tests.test_train_calls_gpu import _model

from magvit2_pytorch_b200._lib import ACT_NONE, SHUFFLE_NONE
from magvit2_pytorch_b200.dist import LfqBatchEntropy
from magvit2_pytorch_b200.train import TapeRunner, TrainRunner

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
STAGE, RESET = "one ring stage missing", "previous tile's accumulators not reset"
CONTROLS = {"dgrad: time taps not flipped", "dgrad: clip i+1 bled into clip i", "SE: last frame gated with the first's gates",
            "entropy: one 32-token block left out", "wgrad: time pad at the back", "wgrad: g one frame late",
            "down-sampler dgrad: pt crop off by one"}


def _lfq_probs64(p, d, inv_t):
    """Per-token code probabilities (N, nc, 2^d) of pre-sign values p (N, nc, d), as _lfq_entropy64 builds them."""
    mask = 2 ** torch.arange(d - 1, -1, -1, device=p.device)
    cb = ((torch.arange(2 ** d, device=p.device)[:, None] & mask) != 0).double() * 2 - 1
    return (2 * inv_t * torch.einsum("tcd,kd->tck", p, cb)).softmax(dim=-1)


def _pt_grad64(x, w, g, k, stride, pad):
    """float64 gradient wrt the time-padded input F.pad(x, pt frames in front) of the conv _conv64_grads takes, uncropped:
    (B, C, pt + T, H, W)."""
    pt, ph, pw = pad
    xp = F.pad(x.double(), (0, 0, 0, 0, pt, 0)).requires_grad_(True)
    with torch.enable_grad():
        y = F.conv3d(F.pad(xp, (pw, pw, ph, ph)), w.double().reshape(w.shape[0], -1, *k), stride=stride)
        gx, = torch.autograd.grad(y, xp, g.double().permute(0, 4, 1, 2, 3))
    return gx


class _Recorder(_BenchRecorder):
    """The benchmark test's recorder on the tokenizer's engine, plus the training step's data gradients, conv backward
    and batch-entropy calls; runners and entropy objects of other engines pass through."""

    def __init__(self, monkeypatch, model):
        super().__init__(monkeypatch, model)
        _, self.table, _ = tokenizer_table()
        self.simt0 = self.eng.simt_conv_calls
        self.nested, self.replaying, self.controls = None, False, {}
        self.bwd, self.n_bwd, self.n_padmode = {}, 0, 0
        self.o_dgrad, self.o_bwd, self.o_pad = TapeRunner._dgrad, TapeRunner._conv_bwd, TrainRunner._conv_bwd_padmode
        self.o_start, self.o_finish = LfqBatchEntropy.start, LfqBatchEntropy.finish
        monkeypatch.setattr(TapeRunner, "_dgrad", self._wrap(self.dgrad, self.o_dgrad))
        monkeypatch.setattr(TapeRunner, "_conv_bwd", self._wrap(self.conv_bwd, self.o_bwd))
        monkeypatch.setattr(TrainRunner, "_conv_bwd_padmode", self._wrap(self.padmode, self.o_pad))
        monkeypatch.setattr(LfqBatchEntropy, "start", self._wrap(self.ent_start, self.o_start))
        monkeypatch.setattr(LfqBatchEntropy, "finish", self._wrap(self.ent_finish, self.o_finish))

    def _wrap(self, mine, orig):
        rec = self

        def wrapped(obj, *a, **k):
            if obj.eng is not rec.eng or rec.replaying:
                return orig(obj, *a, **k)
            return mine(obj, *a, **k)
        return wrapped

    def _control(self, family, out, wrong, dtype, acc, what):
        """A negative control: the bound rejects the perturbed reference (once per family)."""
        if family not in self.controls:
            _rejects(out, wrong, dtype, acc, f"{what}: {family}")
            self.controls[family] = what

    # ---------------------------------------------------------------- the table of tests/test_train_calls_cpu.py
    def _roles(self):
        """{id(pack): role} of the tokenizer's forward convs."""
        m, P = self.m, self.eng._packs
        roles = {id(P["conv_in_tc"]): "conv_in_kw", id(P["conv_out"]): "conv_out"}
        for side, stages in (("enc", m.stages), ("dec", list(reversed(m.stages)))):
            for i, st in enumerate(stages):
                key = f"{side}{i}"
                if st.kind == "residual":
                    for j in range(st.count):
                        roles[id(P[f"{key}.{j}"]["conv3"])], roles[id(P[f"{key}.{j}"]["conv1"])] = "conv3", "conv1"
                elif st.kind in ("compress_space", "compress_time"):
                    roles[id(P[key])] = ("down_" if side == "enc" else "up_") + st.kind.split("_")[1]
                else:
                    a, ff = P[key + ".attn"], P[key + ".ff"]
                    roles.update({id(a[k]): k for k in ("q", "kv", "qkv") if k in a})
                    roles.update({id(a["out"]): "attn_out", id(ff["fc1"]): "fc1", id(ff["fc2"]): "fc2"})
        return roles

    def _table(self, rec, role, x_shape, Co):
        key = ("tok", role, tuple(x_shape), Co)
        want, block = self.table.get(key, (None, None))
        assert want is not None, f"call {len(self.calls)}: {key} is not in the table of tests/test_train_calls_cpu.py"
        assert rec["kind"] == want, f"call {len(self.calls)}: {key} ran {rec['kind']}, the table says {want}"
        if rec["kind"] == "simt":
            assert ("tok", role, block) in TOK_SIMT_BY_DESIGN, f"{key}: a bf16 call fell back to the CUDA-core conv"
        rec.update(key=key, role=role)

    # ---------------------------------------------------------------- Engine.conv
    def conv(self, x, pk, **kw):
        if self.replaying:
            return self.orig["conv"](x, pk, **kw)
        if self.nested is not None:         # the transposed conv of a data gradient: the dgrad wrapper checks it
            kind, y = _ran(self.eng, lambda: self.orig["conv"](x, pk, **kw))
            self.nested.update(kind=kind, pk=pk, ta=self.eng._tc_args(x, pk, pad=kw.get("pad"),
                                                                      out_spatial=kw.get("out_spatial"), y=y))
            return y
        n = len(self.calls)
        role = self._roles().get(id(pk))
        assert role is not None, f"call {n}: a conv with a pack the tokenizer does not own"
        y = super().conv(x, pk, **kw)
        self._table(self.calls[n], role, x.shape, pk.Co)
        return y

    def _check_conv(self, rec, x, y, what, exact=False, w=None, b=None, res=None, video=None, defects=False, os=None):
        super()._check_conv(rec, x, y, what, exact=exact, w=w, b=b, res=res, video=video, os=os)
        if defects and rec["kind"] == "slab" and rec["pk"].epi_mode == 0 and rec["shuffle"] == SHUFFLE_NONE and \
                not rec["conv_in"]:
            xs, w, b, kw = self._conv_ref_args(rec, video if rec["conv_in"] else x, w, b)
            rec["rejected"] = self._defects(rec, xs, w, b, y, kw, res)

    def _defects(self, rec, xs, w, b, y, kw, res):
        """_defect_deltas at the schedule's last tile, each rejected by the exact bound.  A data gradient reads frames
        t .. t + kt - 1, so at the clip's last frame its missing ring stage is frame tap 0's."""
        deltas = _defect_deltas(self.lib, rec["ta"], self.n_sm, xs, w, kw["pad"], kw["out_sp"], kw.get("tp"), rec["plan"])
        for defect, (i, delta) in deltas.items():
            r = None if res is None else res[i:i + 1].double()
            ref, acc = forward64(xs(i), w, b, None, r, dtype=BF, exact=True, **kw)
            wrong, _ = forward64(xs(i), w, b, None, r, dtype=BF, exact=True, delta=delta, **kw)
            _rejects(y[i:i + 1], wrong, BF, acc, f"{rec['key']}: {defect}")
        return sorted(deltas)

    # ---------------------------------------------------------------- SqueezeExcite
    def squeeze_excite_residual(self, y, x, p):
        n0 = len(self.guard.allocs)
        out = self.orig["squeeze_excite_residual"](y, x, p)
        what = f"call {len(self.calls)}: squeeze_excite_residual {tuple(x.shape)}"
        torch.cuda.synchronize()
        B, T, H, W, C_ = x.shape
        gates = self._alloc(n0 + 1, (B * T, C_))
        self._check_gates(x, y, gates, out, p, what)
        wg = gates.double().reshape(B, T, C_).clone()
        wg[:, -1] = wg[:, 0]
        gr = (wg.reshape(B * T, 1, C_) * y.double().reshape(B * T, H * W, C_) + x.double().reshape(B * T, H * W, C_))
        self._control("SE: last frame gated with the first's gates", out.reshape(B * T, H * W, C_), gr, BF, U * gr.abs(),
                      what)
        self._done(n0, what)
        self.calls.append(dict(op="se", kind="simt", C=C_))
        return out

    # ---------------------------------------------------------------- LFQ batch entropy
    def ent_start(self, be, presign, group=None):
        self.o_start(be, presign, group)
        self.presign = presign

    def ent_finish(self, be, diversity_gamma=2.5, entropy_w=0.1, commit_w=1.0, group=None):
        avg, stats, N, d = be._pending
        out = self.o_finish(be, diversity_gamma, entropy_w, commit_w, group)
        torch.cuda.synchronize()
        what = f"call {len(self.calls)}: batch entropy N {N} d {d}"
        nc, inv_t = be.nc, be.inv_temperature
        p = self.presign.double().reshape(N, nc, d)
        nblk = -(-N // 32)
        # the logits' rounding (module docstring): each probability of token t within a factor 1 +- D_t
        e = 1.001 * (d + 2) * U * 2 * inv_t * p.abs().sum(dim=-1)                    # (N, nc)
        D = torch.expm1(2 * e)
        prob = _lfq_probs64(p, d, inv_t)
        h_t = (-prob * torch.log(prob.clamp(min=1e-300))).sum(dim=-1)
        e_ent = (D * (h_t + 1 + 2 * e)).sum().item()
        e_avg = torch.einsum("tc,tck->ck", D, prob).reshape(-1) / N
        del prob, h_t

        def check(p_, avg_, stats_, err_ent, err_avg):
            """-> the names of the outputs outside their bounds."""
            ent, com, prob_sum = _lfq_entropy64(p_, d, inv_t)
            rel = (2 ** d // 256 + 80 + 8 * nblk) * U
            bad = []
            if abs(stats_[0].item() - ent.item()) > rel * (ent.item() + N * nc) + err_ent:
                bad.append("entropy sum")
            if abs(stats_[1].item() - com.item()) > (d + 40 + nblk) * U * com.item():
                bad.append("commitment sum")
            want = prob_sum.reshape(-1) / N
            if ((avg_.double() - want).abs() > (rel + U) * want + err_avg + 1e-36 * N).any():
                bad.append("avg_prob")
            return bad, ent, com, want

        bad, ent, com, avg64 = check(p, avg, stats, e_ent, e_avg)
        assert not bad, f"{what}: {bad} outside their bounds"
        # one 32-token block (the middle one) left out
        j = nblk // 2
        keep = torch.ones(N, dtype=torch.bool, device=p.device)
        keep[32 * j:32 * (j + 1)] = False
        bad_w, _, _, _ = check(p[keep], avg, stats, e_ent, e_avg)
        assert bad_w, f"{what}: the bound does not reject one 32-token block left out"
        self.controls["entropy: one 32-token block left out"] = f"{what}: rejected by {bad_w}"
        # mv2_lfq_aux_finalize on the kernel's avg_prob and stats, against float64
        ps, cm = ent.item() / (N * nc), com.item() / (N * nc * d)
        be64 = (-avg64 * torch.log(avg64.clamp(min=1e-5))).reshape(nc, -1).sum(dim=-1).mean().item()
        aux = (ps - diversity_gamma * be64) * entropy_w + cm * commit_w
        scale = [abs(ps), abs(be64), abs(cm), entropy_w * (abs(ps) + diversity_gamma * abs(be64)) + commit_w * abs(cm)]
        for k, (got, want) in enumerate(zip(out, (ps, be64, cm, aux))):
            assert abs(got.item() - want) <= 1e-4 * scale[k] + 1e-6, (what, k, got.item(), want)
        self.calls.append(dict(op="entropy", kind="simt", N=N))
        return out

    # ---------------------------------------------------------------- data gradients
    def dgrad(self, runner, g, w, k, out_spatial):
        n0 = len(self.guard.allocs)
        self.nested = inner = {}
        try:
            out = self.o_dgrad(runner, g, w, k, out_spatial)
        finally:
            self.nested = None
        what = f"call {len(self.calls)}: dgrad k{k} g {tuple(g.shape)} on {inner.get('kind')}"
        self._done(n0, what)
        rec = dict(op="dgrad", kind=inner["kind"], pk=inner["pk"], ta=inner["ta"], x_shape=tuple(g.shape),
                   w_shape=tuple(w.shape), k=tuple(k), out_sp=tuple(out_spatial), runner=runner)
        self._table(rec, f"dgrad k{''.join(map(str, k))}", g.shape, w.shape[1])
        if rec["kind"] == "slab":
            rec["plan"] = _lib_plan(self.lib, inner["ta"], self.n_sm)
        self._check_dgrad(rec, g, w, out, what, controls=True)
        self.calls.append(rec)
        return out

    def _check_dgrad(self, rec, g, w, out, what, exact=False, controls=False):
        k, osp = rec["k"], rec["out_sp"]
        K = w.shape[0] * math.prod(k)
        for i in range(g.shape[0]):
            gi = g[i:i + 1]
            ref = _dgrad64(gi, w, k, osp)
            acc = 0 if exact else _gamma(K, C_OF[rec["kind"]]) * _dgrad64(gi.abs(), w.abs(), k, osp)
            _check(out[i:i + 1], ref, out.dtype, acc, f"{what}, clip {i}")
            if controls and i == 0 and k[0] > 1 and g[1, :2].abs().max() > 0:
                self._control("dgrad: time taps not flipped", out[:1], _dgrad64(gi, w.flip(2), k, osp), out.dtype, acc,
                              what)
                if "dgrad: clip i+1 bled into clip i" not in self.controls:
                    T = osp[0]
                    bled = _dgrad64(g[:2].reshape(1, 2 * T, *g.shape[2:]), w, k, (2 * T,) + osp[1:])[:, :T]
                    self._control("dgrad: clip i+1 bled into clip i", out[:1], bled, out.dtype, acc, what)
            del ref, acc

    # ---------------------------------------------------------------- weight / strided data gradients
    def padmode(self, runner, g, x, weight, bias, k, pad_mode, need_gx=True):
        assert pad_mode == "constant", pad_mode        # the README tokenizer's conv_out: _conv_bwd_padmode delegates
        self.n_padmode += 1
        return self.o_pad(runner, g, x, weight, bias, k, pad_mode, need_gx)

    def conv_bwd(self, runner, g, x, weight, bias, k, stride=(1, 1, 1), pad=None, need_gx=True, x_is_cf=False):
        out = self.o_bwd(runner, g, x, weight, bias, k, stride, pad, need_gx, x_is_cf)
        self.n_bwd += 1
        key = (tuple(g.shape), tuple(x.shape), tuple(x.stride()), tuple(weight.shape), bias is not None, tuple(k),
               tuple(stride), None if pad is None else tuple(pad), need_gx, x_is_cf)
        self.bwd.setdefault(key, dict(runner=runner, n=0))["n"] += 1
        return out

    def replay_bwd(self, key, runner, gen):
        """The _conv_bwd call `key` again through the same method, on operands in {-1, 0, 1}; -> the controls it ran."""
        g_shape, x_shape, x_stride, w_shape, has_b, k, stride, pad, need_gx, x_is_cf = key

        def t(shape):
            return torch.randint(-1, 2, shape, generator=gen, device="cuda").double()
        g, w, b, x64 = t(g_shape), t(w_shape), t(w_shape[:1]), t(x_shape)
        if not has_b:
            b = torch.zeros_like(b)
        x = torch.empty_strided(x_shape, x_stride, device="cuda", dtype=BF).copy_(x64)
        W = torch.nn.Parameter(w.to(BF))
        Bp = torch.nn.Parameter(b.to(BF)) if has_b else None
        n0 = len(self.guard.allocs)
        grads, runner.grads = runner.grads, {}
        self.replaying = True
        try:
            gx = self.o_bwd(runner, g.to(BF).contiguous(), x, W, Bp, k, stride, pad, need_gx, x_is_cf)
            gw, gb = runner.grads.get(W), runner.grads.get(Bp) if has_b else None
        finally:
            runner.grads, self.replaying = grads, False
        what = f"replay of _conv_bwd g {g_shape} x {x_shape} k {k} stride {stride} pad {pad} need_gx {need_gx} cf {x_is_cf}"
        self._done(n0, what)
        kt, kh, kw = k
        pad_ = pad if pad is not None else (kt - 1, kh // 2, kw // 2)
        x_cf = x64 if x_is_cf else x64.permute(0, 4, 1, 2, 3)
        rgx, rgw, rgb = _conv64_grads(x_cf, w, b, g, k, stride, pad_)
        _check(gw, rgw, BF, 0, f"{what}: weight gradient")
        if has_b:
            _check(gb, rgb, BF, 0, f"{what}: bias gradient")
        if need_gx:
            _check(gx, rgx if x_is_cf else rgx.permute(0, 2, 3, 4, 1), BF, 0, f"{what}: data gradient")
        else:
            assert gx is None
        del rgx, rgb
        if pad_[0] > 0 and "wgrad: time pad at the back" not in self.controls:
            _, wgw, _ = _conv64_grads(x_cf, w, b, g, k, stride, pad_, back=True)
            self._control("wgrad: time pad at the back", gw, wgw, BF, 0, what)
        if "wgrad: g one frame late" not in self.controls:
            g_late = torch.zeros_like(g)
            g_late[:, 1:] = g[:, :-1]
            _, wgw, _ = _conv64_grads(x_cf, w, b, g_late, k, stride, pad_)
            self._control("wgrad: g one frame late", gw, wgw, BF, 0, what)
        own = pad is None and tuple(stride) == (1, 1, 1) and not x_is_cf
        if need_gx and not own and pad_[0] > 0 and "down-sampler dgrad: pt crop off by one" not in self.controls:
            gxp = _pt_grad64(x_cf, w, g, k, stride, pad_)
            wrong = gxp[:, :, pad_[0] - 1:-1].permute(0, 2, 3, 4, 1)
            self._control("down-sampler dgrad: pt crop off by one", gx, wrong, BF, 0, what)

    # ---------------------------------------------------------------- exact replay of the wgmma calls
    def replay_dgrad(self, rec, gen):
        g, w = _grid(rec["x_shape"], "x", gen), _grid(rec["w_shape"], "w", gen)
        n0 = len(self.guard.allocs)
        self.nested = inner = {}
        try:
            out = self.o_dgrad(rec["runner"], g.to(BF).contiguous(), w.to(BF), rec["k"], rec["out_sp"])
        finally:
            self.nested = None
        what = f"replay of {rec['key']}"
        self._done(n0, what)
        assert inner["kind"] == rec["kind"], f"{what}: ran {inner['kind']}"
        self._check_dgrad(rec, g, w, out, what, exact=True)
        if rec["kind"] != "slab":
            return []
        pk, k = inner["pk"], rec["k"]        # the transposed conv the kernel ran, for the defects' accumulators
        wt = pk.w.double().permute(2, 1, 0).reshape(pk.Co, pk.Ci, *pk.k)
        kw = dict(kern="slab", stride=(1, 1, 1), pad=(0, k[1] // 2, k[2] // 2), out_sp=rec["out_sp"],
                  K=math.prod(pk.k) * pk.Ci, act=ACT_NONE, mode=0)
        return self._defects(dict(rec, ta=inner["ta"]), lambda i: g[i:i + 1], wt,
                             torch.zeros(pk.Co, device="cuda", dtype=torch.float64), out, kw, None)


def test_readme_train_step_tokenizer_calls_vs_float64(monkeypatch):
    t0 = time.time()
    m = _model()
    video = synth_data.synth_video(CLIPS, 3, FRAMES, 128).cuda().bfloat16()
    torch.manual_seed(1)                  # the frame picks draw from torch's CPU generator
    loss, _ = m(video, return_loss=True)  # warm-up: the discriminator's and the VGG's packs and engines
    loss.backward()
    del loss
    rec = _Recorder(monkeypatch, m)
    torch.manual_seed(2)
    loss, _ = m(video, return_loss=True)
    loss.backward()
    del loss
    torch.cuda.synchronize()
    calls, eng = rec.calls, rec.eng
    # ---- structure: calls per kind, kernels, tiles per CTA, negative controls of part 1 ----
    got = {op: sum(c["op"] == op for c in calls) for op in ("conv", "se", "rmsnorm", "dgrad", "quantize", "entropy")}
    got.update(conv_bwd=rec.n_bwd, padmode=rec.n_padmode)
    want = tokenizer_counts(m)
    print(f"\ncalls checked per kind {got}")
    assert got == want, f"calls per kind {got}, the module structure implies {want}"
    assert not any(c["op"] in ("ru", "codes") for c in calls)
    seen = {c["key"] for c in calls if "key" in c}
    assert seen == set(rec.table), (set(rec.table) - seen, seen - set(rec.table))
    assert eng.simt_conv_calls - rec.simt0 == sum(c["kind"] == "simt" and c["op"] in ("conv", "dgrad") for c in calls)
    big = [c for c in calls if c.get("role") in ("conv3", "conv1", "dgrad k333", "dgrad k111") and c["kind"] == "slab" and
           c["x_shape"][2] == 128]
    assert len(big) == 8 and all(c["plan"]["total"] > 2 * c["plan"]["grid"] for c in big), [c.get("plan") for c in big]
    # ---- part 2: exact replay of every distinct wgmma call, the pipeline defects ----
    gen = torch.Generator(device="cuda").manual_seed(7)
    rejected = {}
    for c in calls:
        if c["op"] not in ("conv", "dgrad") or c["kind"] == "simt":
            continue
        key = ("conv", _replay_key(c)) if c["op"] == "conv" else ("dgrad", c["key"], c["k"], c["out_sp"])
        if key in rejected:
            continue
        if c["op"] == "conv":
            rec.replay(c, gen, defects=True)
            got_d = sorted(c.pop("rejected", []))
        else:
            got_d = rec.replay_dgrad(c, gen)
        rejected[key] = (c, got_d)
    n_def = 0
    for key, (c, got_d) in rejected.items():
        plain = c["op"] == "dgrad" or (c["kind"] == "slab" and c["pk"].epi_mode == 0 and c["shuffle"] == SHUFFLE_NONE and
                                       not c["conv_in"])
        assert got_d == (sorted([STAGE, RESET]) if plain else []), (c["key"], got_d)
        n_def += plain
    for role, shape in (("conv3", (CLIPS, 20, 128, 128, 64)), ("conv1", (CLIPS, 20, 128, 128, 64)),
                        ("dgrad k333", (CLIPS, 20, 128, 128, 64)), ("dgrad k111", (CLIPS, 20, 128, 128, 64)),
                        ("dgrad k333", (CLIPS, 20, 16, 16, 512))):
        assert any(c["key"][1:3] == (role, shape) and got_d for c, got_d in rejected.values()), (role, shape)
    # ---- part 3: the weight and strided data gradients, replayed through _conv_bwd ----
    cost = lambda kv: math.prod(kv[0][0]) * math.prod(kv[0][3])        # noqa: E731
    for key, r in sorted(rec.bwd.items(), key=cost):
        rec.replay_bwd(key, r["runner"], gen)
    rec._done(0, "allocations outside the checked calls")
    assert set(rec.controls) == CONTROLS, set(rec.controls) ^ CONTROLS
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"{len(rejected)} distinct wgmma calls replayed exactly, {n_def} of them rejecting both pipeline defects; "
          f"{len(rec.bwd)} distinct _conv_bwd calls replayed exactly; controls rejected: {sorted(rec.controls.items())}; "
          f"wall {time.time() - t0:.0f} s, peak device memory {peak:.1f} GiB")
