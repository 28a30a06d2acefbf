"""Every conv-path kernel call of the benchmark's step (tokenize, then decode_from_code_indices) at the benchmark's own
shapes, checked one call at a time against float64.

The workloads are built as bench.py builds them (its README_KW / WORKLOADS / FRAMES, synth_data weights, bf16, eval):
  * readme: 4 clips of 3 x 17 x 128 x 128 (the benchmark's batch 0);
  * cfg4:   256^2, max_dim = 1024, one clip instead of the benchmark's 3 (it still reaches the 1024-channel layers).

Part 1, real data.  The engine's entry points are wrapped on the instance.  Each call is checked right after it returns
(synchronise, float64 reference from the call's own bf16 operands one clip at a time, check, free), so the peak memory
stays near one layer's float64 tensors.  The engine's allocator is wrapped as in tests/test_conv_forward_gpu.py: every
output starts NaN-filled between two sentinels, checked when the call returns.  References and bounds are the ones of
the kernel tests, reused:
  * Engine.conv (slab, down-space, tap-wise, the kw-packed conv_in, the channels-first conv_out, GEGLU, shuffles,
    residuals, the time-strided slab): forward64 / geglu64 of tests/test_conv_forward_gpu.py.  The weights come from the
    module (conv_in) or from pk.w, the CUDA-core layout, so the wgmma repackings (pack_ff's row pairing, the shuffle row
    order, pack_conv_down_space, the kw packing) are checked with the kernel;
  * Engine.residual_unit, fused: y by ru_y64 (with the bf16 rounding-boundary rule for h), the SE gates against
    _se_gates64 of the kernel's own y within GATE_TOL, then gate_residual; unfused: its two convs as above, then
    squeeze_excite_residual the same way;
  * Engine.rmsnorm: test_simt_ops_gpu's _rms_ref bound;
  * quantize_cl / codes_to_quantized_cl: test_simt_ops_gpu.test_lfq's reference; indices exact except where the float64
    pre-sign value lies within its allowance of zero.
The attention kernels themselves are checked call by call in tests/test_attention_gpu.py and are left out.  The test
asserts the number of calls of each kind the stages imply, which kernel ran each call (no bf16 call on the CUDA-core
conv), and, from mv2_tc_slab_plan with the device's SM count, that each slab flavour ran at least one call with more than
two tiles per CTA, so every CTA carried its rings and accumulator staging from one tile into the next.

Part 2, exact replay.  At real-data depths (K up to 27 x 1024) the rigorous per-element accumulation allowance is larger
than one missing K-chunk's contribution.  So every distinct wgmma conv call (and fused ResidualUnit) is replayed with the
same entry point, shapes, arguments and packer on operands from a dyadic grid (REPLAY_GRID): every product and partial
sum is then a multiple of 2^-8 below 2^14, so the fp32 accumulation is exact in any order, even with an adder that
truncates, and the allowance is the epilogue's alone (the fused RU's 1x1x1 GEMM reads bf16-rounded h and keeps its own).
On the fused RU, on a 512- / 1024-channel EPI_PLAIN conv and on conv_out the bound must reject two pipeline defects at
the schedule's last tile (mv2_tc_slab_tile): one ring stage (frame tap x 64-channel K-chunk x in-plane tap) missing,
and the accumulators of the CTA's previous tile not reset.

Part 3, launch mode.  The benchmark runs the step through StreamLanes(model, 3) with CUDA graphs, with and without
programmatic dependent launch.  Nine steps on distinct batches (plain call, capture and replay on every lane) must equal
the eager outputs bit for bit, and the eager step of batch 0 must equal what part 1 checked."""
import ctypes as C
import math

import pytest
import torch

import synth_data
from bench import FRAMES, WORKLOADS
from oracle import restated as R
from tests.test_conv_forward_gpu import HEAD, _conv64, _Guard, _ran, forward64, geglu64, ru_y64
from tests.test_simt_ops_gpu import GATE_TOL, U, _check, _proj_err, _quant_sd, _rejects, _rms_ref, _se_gates64

from magvit2_pytorch_b200 import StreamLanes, VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_ELU, ACT_NONE, SHUFFLE_NONE, SHUFFLE_SPACE, SHUFFLE_TIME
from magvit2_pytorch_b200.engine import pack_conv, pack_conv_down_space, pack_conv_in_kwpack, pack_ff

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
# the replay grid: x, residual and video in {-8..8} / 2^2, weights in {-8..8} / 2^6, biases in {-64..64} / 2^8; a conv's
# per-clip oscale (the Conv3DMod's demodulation) in {1..8} / 2^3
REPLAY_GRID = dict(x=(8, 2), w=(8, 6), b=(64, 8), os=(8, 3))
FLAVOURS = ("ru_c64", "ru_c128", "plain", "plain_res", "geglu", "down", "time_stride", "shuffle", "ragged_cf", "conv_in")
_EAGER = {}          # workload -> (codes, reconstruction) of the checked eager step, for the launch-mode test


def _workload(name):
    wl = WORKLOADS[name]
    torch.manual_seed(0)
    model = VideoTokenizer(**wl["kw"])
    synth_data.fill_state_dict_(model, 0)
    model = model.cuda().bfloat16().eval()
    clips = wl["clips"] if name == "readme" else 1
    return model, clips, wl["size"]


def _grid(shape, which, gen):
    n, e = REPLAY_GRID[which]
    v = torch.randint(-n, n + 1, shape if isinstance(shape, tuple) else (shape,), generator=gen, device="cuda")
    return v.double() * 2.0 ** -e


def _n_sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _lib_plan(lib, ta, n_sm):
    out = (C.c_int32 * 6)()
    assert lib.mv2_tc_slab_plan(C.byref(ta), n_sm, out) == 0, lib.mv2_last_error()
    return dict(zip(("mw", "bn", "n_tiles_n", "total", "grid", "slab_stages"), out))


def last_cta(total, grid):
    """The CTA that runs the schedule's last tile (tc_slab.cu slab_tile_of_cta: waves alternate direction)."""
    k, r = divmod(total - 1, grid)
    return grid - 1 - r if k & 1 else r


def _last_tiles(lib, ta, n_sm):
    """(previous, last) tile (tile, b, t, h0, w0, n0) of the CTA that runs the schedule's last tile."""
    plan = _lib_plan(lib, ta, n_sm)
    cta = last_cta(plan["total"], plan["grid"])
    out, k, tiles = (C.c_int32 * 6)(), 0, []
    while True:
        assert lib.mv2_tc_slab_tile(C.byref(ta), n_sm, cta, k, out) == 0, lib.mv2_last_error()
        if out[0] < 0:
            assert tiles[-1][0] == plan["total"] - 1 and len(tiles) >= 2, tiles
            return tiles[-2], tiles[-1]
        tiles.append(tuple(out))
        k += 1


def _region(tile, plan, shape):
    """Index of one tile's outputs in a (1, To, Ho, Wo, Co) accumulator.  The accumulators are channels-last whatever the
    output's layout: a channels-first output (out_layout 1) compares with them permuted to (1, Co, To, Ho, Wo)."""
    _, _, t, h0, w0, n0 = tile
    _, To, Ho, Wo, Co = shape
    return (0, t, slice(h0, min(h0 + 16, Ho)), slice(w0, min(w0 + 8 * plan["mw"], Wo)), slice(n0, min(n0 + plan["bn"], Co)))


def _acc64(x, w, pad, out_sp, tp):
    """The conv's accumulators (no bias) as forward64 builds them: stride 1, tp leading output frames dropped.  With tp None
    the leading time pad may be negative: the transposed conv of a data gradient with its first -pad[0] output frames
    cropped (output frame t reads input frames t - pad[0] ..)."""
    if tp is None:
        return _conv64(x, w, (1, 1, 1), pad, out_sp)
    kt = w.shape[2]
    return _conv64(x, w, (1, 1, 1), (kt - 1,) + tuple(pad[1:]), (x.shape[1],) + tuple(out_sp[1:]))[:, tp:]


def _defect_deltas(lib, ta, n_sm, xs, w, pad, out_sp, tp, plan):
    """{defect: (clip, delta)} at the schedule's last tile: one ring stage (the centre in-plane tap, input channels 0..63,
    of the last frame tap that reads inside the clip at that tile's frame) missing, and the previous tile's accumulators
    added.  xs(b) gives clip b's float64 operand.  Output frame t reads input frames t - pad[0] + d (pad[0] = kt - 1 - tp
    for a conv with tp cropped frames): a causal conv's last frame reads its last frame at tap kt - 1, a data gradient's
    (the transposed conv, pad[0] <= 0) only at tap 0."""
    prev, last = _last_tiles(lib, ta, n_sm)
    b = last[1]
    kt, kh, kw = w.shape[2:]
    ft = min(kt - 1, xs(b).shape[1] - 1 - last[2] + pad[0])
    assert ft >= 0, (last, pad)
    ws = torch.zeros_like(w)
    ws[:, :64, ft, kh // 2, kw // 2] = w[:, :64, ft, kh // 2, kw // 2]
    stage = _acc64(xs(b), ws, pad, out_sp, tp)
    r = _region(last, plan, stage.shape)
    d_stage = torch.zeros_like(stage)
    d_stage[r] = -stage[r]
    acc_prev = _acc64(xs(prev[1]), w, pad, out_sp, tp)
    rp = _region(prev, plan, acc_prev.shape)
    d_reset = torch.zeros_like(stage)
    a, p_ = d_reset[r], acc_prev[rp]
    n = [min(u, v) for u, v in zip(a.shape, p_.shape)]
    d_reset[r][:n[0], :n[1], :n[2]] = p_[:n[0], :n[1], :n[2]]
    assert (prev[2:] != last[2:] or prev[1] != b) and d_reset.abs().max() > 0 and d_stage.abs().max() > 0
    return {"one ring stage missing": (b, d_stage), "previous tile's accumulators not reset": (b, d_reset)}


class _Recorder:
    """Wraps the entry points of one engine; every call is checked when it returns (module docstring)."""

    def __init__(self, monkeypatch, model):
        self.m, self.eng = model, model.engine
        eng = self.eng
        self.lib, self.n_sm = eng.lib, _n_sm()
        self.guard = _Guard(eng)
        self.calls, self.ingest = [], None
        self.orig = {k: getattr(eng, k) for k in ("conv", "residual_unit", "squeeze_excite_residual", "rmsnorm",
                                                   "quantize_cl", "codes_to_quantized_cl", "ingest_kwpack")}
        monkeypatch.setattr(eng, "_new", self.guard.new)
        monkeypatch.setattr(eng, "conv_log", [])
        for k in self.orig:
            monkeypatch.setattr(eng, k, getattr(self, k))

    # ---------------------------------------------------------------- allocations
    def _done(self, n0, what):
        """The borders of the allocations made since n0 unchanged; then they are no longer tracked."""
        torch.cuda.synchronize()
        for i, (buf, n, head, tail) in enumerate(self.guard.allocs[n0:]):
            assert torch.equal(buf[:HEAD], head), f"{what}: store before allocation {i}"
            assert torch.equal(buf[HEAD + n:], tail), f"{what}: store past the end of allocation {i}"
        del self.guard.allocs[n0:]

    def _alloc(self, i, shape):
        buf, n = self.guard.allocs[i][:2]
        return buf[HEAD:HEAD + n].view(shape)

    # ---------------------------------------------------------------- Engine.conv
    def ingest_kwpack(self, v, t_pad, pin):
        self.ingest = (v, t_pad)
        return self.orig["ingest_kwpack"](v, t_pad, pin)

    def conv(self, x, pk, **kw):
        n0 = len(self.guard.allocs)
        kind, y = _ran(self.eng, lambda: self.orig["conv"](x, pk, **kw))
        what = f"call {len(self.calls)}: conv {kind} x {tuple(x.shape)} -> {tuple(y.shape)}"
        self._done(n0, what)
        rec = self._conv_record(x, pk, kw, y, kind)
        self._check_conv(rec, x, y, what, res=kw.get("res"), video=self.ingest[0] if rec["conv_in"] else None,
                         os=kw.get("oscale"))
        self.calls.append(rec)
        return y

    def _conv_record(self, x, pk, kw, y, kind):
        assert not kw.get("token_shift") and kw.get("ss") is None
        kt, kh, kw_ = pk.k_tc or pk.k
        d = dict(op="conv", kind=kind, pk=pk, x_shape=tuple(x.shape), y_shape=tuple(y.shape), os=kw.get("oscale") is not None,
                 stride=tuple(kw.get("stride", (1, 1, 1))), act=kw.get("act", ACT_NONE),
                 shuffle=kw.get("shuffle", SHUFFLE_NONE), res=kw.get("res") is not None, out_cf=bool(kw.get("out_cf")),
                 pad=tuple(kw.get("pad") or (kt - 1, kh // 2, kw_ // 2)),
                 out_sp=tuple(kw.get("out_spatial") or x.shape[1:4]))
        d["conv_in"] = pk is self.eng._packs.get("conv_in_tc")
        if d["conv_in"]:
            d["t_pad"] = self.ingest[1]
        ta = self.eng._tc_args(x, pk, d["stride"], d["pad"], d["out_sp"], d["act"], d["shuffle"], d["out_cf"],
                               res=kw.get("res"), y=y, oscale=kw.get("oscale"))
        d["ta"] = ta
        if kind == "slab":
            d["plan"] = _lib_plan(self.lib, ta, self.n_sm)
            d["flavour"] = ("conv_in" if d["conv_in"] else "geglu" if pk.epi_mode == 1 else
                            "shuffle" if d["shuffle"] != SHUFFLE_NONE else "ragged_cf" if d["out_cf"] else
                            "time_stride" if d["stride"] == (2, 1, 1) else "plain_res" if d["res"] else "plain")
        elif kind == "down":      # no plan entry point: the tile count with the widest macro tile (mw = 4) bounds it below
            B, To, Ho, Wo = x.shape[0], *d["out_sp"]
            bn = next(c for c in (128, 64, 32) if pk.Co_tc % c == 0)
            total = B * To * -(-Ho // 16) * -(-Wo // 32) * (pk.Co_tc // bn)
            d["plan"] = dict(total=total, grid=min(total, self.n_sm))
            d["flavour"] = "down"
        else:
            d["flavour"] = kind
        return d

    def _conv_ref_args(self, rec, x, w=None, b=None):
        """(per-clip operand function, w, b, forward64 keywords) of a recorded call; w / b default to the call's own."""
        pk = rec["pk"]
        if rec["conv_in"]:        # the video (rounded to bf16 as mv2_ingest_kwpack reads it) and the module's weight
            video = x
            if w is None:
                w, b = self.m.conv_in.conv.weight.double(), self.m.conv_in.conv.bias.double()
            tp_ = rec["t_pad"]
            xs = lambda i: torch.nn.functional.pad(video[i:i + 1].to(BF).double().permute(0, 2, 3, 4, 1),
                                                   (0, 0, 0, 0, 0, 0, tp_, 0))
            kt, kh, kw_ = w.shape[2:]
            return xs, w, b, dict(kern="slab", stride=(1, 1, 1), pad=(kt - 1, kh // 2, kw_ // 2), out_sp=rec["out_sp"],
                                  K=kt * kh * 32, act=rec["act"])
        if w is None:
            w = pk.w.double().permute(2, 1, 0).reshape(pk.Co, pk.Ci, *pk.k)
            b = pk.bias.double() if pk.bias is not None else torch.zeros(pk.Co, device="cuda", dtype=torch.float64)
        xs = lambda i: x[i:i + 1, ..., :pk.Ci].double()
        kt = pk.k[0]
        tp = (kt - 1) - rec["pad"][0] if rec["out_cf"] else None
        K = 12 * pk.Ci if rec["kind"] == "down" else math.prod(pk.k) * pk.Ci
        return xs, w, b, dict(kern=rec["kind"], stride=rec["stride"], pad=rec["pad"], out_sp=rec["out_sp"], K=K,
                              act=rec["act"], mode=pk.epi_mode, shuffle=rec["shuffle"], tp=tp)

    def _check_conv(self, rec, x, y, what, exact=False, w=None, b=None, res=None, video=None, defects=False, os=None):
        """os: the call's per-clip oscale (B, Co), or None.  A call on the CUDA-core conv fails unless its record names it
        as meant to run there (simt_ok)."""
        pk, B = rec["pk"], rec["x_shape"][0]
        assert rec["kind"] != "simt" or rec.get("simt_ok"), f"{what}: a bf16 conv fell back to the CUDA-core kernel"
        osc = (lambda i: None) if os is None else (lambda i: os[i:i + 1].double())
        if pk.epi_mode == 1:      # fc1 + GEGLU; the hidden channels pack_ff pads in are exactly zero
            w1 = pk.w.double()[0].T if w is None else w
            b1 = pk.bias.double() if b is None else b
            I = w1.shape[0] // 2
            assert torch.equal(y[..., I:].float(), torch.zeros_like(y[..., I:].float())), f"{what}: padded channels"
            for i in range(B):
                ref, acc, _ = geglu64(x[i:i + 1].double(), w1, b1, rec["kind"], exact=exact)
                _check(y[i:i + 1, ..., :I], ref, BF, acc, f"{what}, clip {i}")
            return
        xs, w, b, kw = self._conv_ref_args(rec, video if rec["conv_in"] else x, w, b)
        for i in range(B):
            r = None if res is None else res[i:i + 1].double()
            ref, acc = forward64(xs(i), w, b, osc(i), r, dtype=BF, exact=exact, **kw)
            _check(y[i:i + 1], ref, BF, acc, f"{what}, clip {i}")
            del ref
        if defects:
            for defect, (i, delta) in _defect_deltas(self.lib, rec["ta"], self.n_sm, xs, w, kw["pad"], kw["out_sp"],
                                                     kw["tp"], rec["plan"]).items():
                ref, acc = forward64(xs(i), w, b, osc(i), None, dtype=BF, exact=True, **kw)
                wrong, _ = forward64(xs(i), w, b, osc(i), None, dtype=BF, exact=True, delta=delta, **kw)
                _rejects(y[i:i + 1], wrong, BF, acc, f"{what}: {defect}")
                rec.setdefault("rejected", []).append(defect)

    # ---------------------------------------------------------------- ResidualUnit
    def residual_unit(self, x, p, ss=None):
        assert ss is None
        n0, fused0 = len(self.guard.allocs), self.eng.fused_ru_calls
        if p["conv3"].Co not in (64, 128):          # the unfused ResidualUnit: its calls are checked one by one
            out = self.orig["residual_unit"](x, p)
            assert self.eng.fused_ru_calls == fused0
            return out
        kind, out = _ran(self.eng, lambda: self.orig["residual_unit"](x, p))
        assert kind == "ru" and self.eng.fused_ru_calls == fused0 + 1, f"C = {p['conv3'].Co}: ran {kind}, not the fused RU"
        what = f"call {len(self.calls)}: fused RU x {tuple(x.shape)}"
        y = self._alloc(n0, x.shape)
        gates = self._alloc(n0 + 2, (x.shape[0] * x.shape[1], x.shape[-1]))
        rec = self._ru_record(x, p)
        self._check_ru(rec, p, x, y, what)
        self._check_gates(x, y, gates, out, p, what)
        self._done(n0, what)
        self.calls.append(rec)
        return out

    def _ru_record(self, x, p):
        c3 = p["conv3"]
        kt, kh, kw = c3.k
        ta = self.eng._tc_args(x, c3, (1, 1, 1), (kt - 1, kh // 2, kw // 2), tuple(x.shape[1:4]), ACT_ELU, SHUFFLE_NONE,
                               False, y=x)
        C_ = x.shape[-1]
        return dict(op="ru", kind="ru", flavour=f"ru_c{C_}", x_shape=tuple(x.shape), ta=ta,
                    plan=_lib_plan(self.lib, ta, self.n_sm), k=c3.k)

    def _check_ru(self, rec, p, x, y, what, exact=False, w3=None, b3=None, w1=None, b1=None, defects=False):
        c3, c1 = p["conv3"], p["conv1"]
        C_ = x.shape[-1]
        if w3 is None:
            w3 = c3.w.double().permute(2, 1, 0).reshape(C_, C_, *c3.k)
            b3 = c3.bias.double()
            w1 = c1.w.double().permute(2, 1, 0).reshape(C_, C_, 1, 1, 1)
            b1 = c1.bias.double()
        for i in range(x.shape[0]):
            y_ref, ey, _ = ru_y64(x[i:i + 1].double(), w3, b3, w1, b1, exact=exact)
            _check(y[i:i + 1], y_ref, BF, ey, f"{what}: y, clip {i}")
            del y_ref, ey
        if defects:
            kt, kh, kw = c3.k
            xs = lambda i: x[i:i + 1].double()
            for defect, (i, delta) in _defect_deltas(self.lib, rec["ta"], self.n_sm, xs, w3, (kt - 1, kh // 2, kw // 2),
                                                     rec["x_shape"][1:4], None, rec["plan"]).items():
                _, ey, _ = ru_y64(xs(i), w3, b3, w1, b1, exact=True)
                wrong, _, _ = ru_y64(xs(i), w3, b3, w1, b1, exact=True, delta=delta)
                _rejects(y[i:i + 1], wrong, BF, ey, f"{what}: {defect}")
                rec.setdefault("rejected", []).append(defect)

    def _check_gates(self, x, y, gates, out, p, what):
        B, T, H, W, C_ = x.shape
        prm = {k: (p[k] if k == "bk" else p[k].double()) for k in ("wk", "bk", "w1", "b1", "w2", "b2")}
        y_own = y.double().reshape(B * T, H * W, C_)
        err = (gates.double() - _se_gates64(y_own, prm)).abs().max().item()
        assert err <= GATE_TOL, f"{what}: SE gates vs float64 {err:.3g}"
        gr = gates.double()[:, None, :] * y_own + x.double().reshape(B * T, H * W, C_)
        _check(out.reshape(B * T, H * W, C_), gr, BF, U * gr.abs(), f"{what}: gate_residual")

    def squeeze_excite_residual(self, y, x, p):
        n0 = len(self.guard.allocs)
        out = self.orig["squeeze_excite_residual"](y, x, p)
        what = f"call {len(self.calls)}: squeeze_excite_residual {tuple(x.shape)}"
        torch.cuda.synchronize()
        self._check_gates(x, y, self._alloc(n0 + 1, (x.shape[0] * x.shape[1], x.shape[-1])), out, p, what)
        self._done(n0, what)
        self.calls.append(dict(op="se", kind="simt", C=x.shape[-1]))
        return out

    # ---------------------------------------------------------------- norms and the quantiser
    def rmsnorm(self, x, gamma, token_shift=False, ss=None):
        assert ss is None
        n0 = len(self.guard.allocs)
        out = self.orig["rmsnorm"](x, gamma, token_shift)
        what = f"call {len(self.calls)}: rmsnorm {tuple(x.shape)} token shift {token_shift}"
        self._done(n0, what)
        B, T, H, W, C_ = x.shape
        ref = _rms_ref(x.double().reshape(B, T, H * W, C_), gamma.double(), token_shift)
        depth = -(-C_ // 32) + 5
        _check(out.reshape(B, T, H * W, C_), ref, BF, (depth + 6) * U * ref.abs(), what)
        self.calls.append(dict(op="rmsnorm", kind="simt"))
        return out

    def _quant(self):
        qz = self.m.quantizers
        P = self.eng._packs["quant"]
        prm = {k: P[k].double() for k in ("win", "bin", "wout", "bout")}
        return qz, prm, _quant_sd(prm, qz.codebook_dim)

    def quantize_cl(self, x, want_quantized=True, want_aux=False):
        assert not self.m.use_fsq
        n0 = len(self.guard.allocs)
        q, idx, aux = self.orig["quantize_cl"](x, want_quantized, want_aux)
        what = f"call {len(self.calls)}: quantize_cl {tuple(x.shape)}"
        self._done(n0, what)
        qz, prm, sd = self._quant()
        d, nc, C_ = qz.codebook_dim, qz.num_codebooks, x.shape[-1]
        clamp = qz.soft_clamp_input_value
        N = x[..., 0].numel()
        x64 = x.double().reshape(N, C_)
        q_ref, idx_ref, _ = R.lfq_quantize(x64.T.reshape(1, C_, N, 1, 1), sd, clamp if clamp else None, nc, bool(qz.spherical))
        q_ref, idx_ref = q_ref.reshape(C_, N).T, idx_ref.reshape(N, nc)
        lin = x64 @ prm["win"].T + prm["bin"]
        p64 = torch.tanh(lin / clamp) * clamp if clamp else lin
        err = _proj_err(x64, prm) + 4 * U * p64.abs()
        ambiguous = (p64.abs() < err).reshape(N, nc, d).any(dim=-1)
        assert ambiguous.sum().item() <= max(2, N // 100), f"{what}: {ambiguous.sum().item()} ambiguous signs"
        assert torch.equal(idx.reshape(N, nc)[~ambiguous], idx_ref[~ambiguous]), what
        if q is not None:
            acc = (d * nc + 1) * U * (prm["wout"].abs().sum(dim=1) + prm["bout"].abs())
            ok = ~ambiguous.any(dim=1)
            _check(q.reshape(N, C_)[ok], q_ref[ok], BF, acc.expand(N, C_)[ok], f"{what}: quantized")
        if aux is not None and not qz.spherical:
            _check(aux, p64, torch.float32, err, f"{what}: pre-sign values")
        self.calls.append(dict(op="quantize", kind="simt", ambiguous=ambiguous.sum().item(), N=N))
        return q, idx, aux

    def codes_to_quantized_cl(self, codes):
        n0 = len(self.guard.allocs)
        q = self.orig["codes_to_quantized_cl"](codes)
        what = f"call {len(self.calls)}: codes_to_quantized_cl {tuple(codes.shape)}"
        self._done(n0, what)
        qz, prm, sd = self._quant()
        d, nc, C_ = qz.codebook_dim, qz.num_codebooks, q.shape[-1]
        N = math.prod(codes.shape[:4])
        want = R.lfq_indices_to_codes(codes.reshape(N, nc) if nc > 1 else codes.reshape(N), sd, torch.float64, nc)
        acc = (d * nc + 1) * U * (prm["wout"].abs().sum(dim=1) + prm["bout"].abs())
        _check(q.reshape(N, C_), want.reshape(N, C_), BF, acc.expand(N, C_), what)
        self.calls.append(dict(op="codes", kind="simt"))
        return q

    # ---------------------------------------------------------------- exact replay
    def replay(self, rec, gen, defects):
        """The call again, on dyadic-grid operands with the same packer, entry point and arguments (module docstring)."""
        if rec["op"] == "ru":
            return self._replay_ru(rec, gen, defects)
        pk, kind = rec["pk"], rec["kind"]
        x_shape = rec["x_shape"]
        n0 = len(self.guard.allocs)
        kw = dict(stride=rec["stride"], pad=rec["pad"], out_spatial=rec["out_sp"], act=rec["act"], shuffle=rec["shuffle"],
                  out_cf=rec["out_cf"])
        video = res = None
        if rec["conv_in"]:
            w, b = _grid(tuple(self.m.conv_in.conv.weight.shape), "w", gen), _grid(pk.Co, "b", gen)
            pk2 = pack_conv_in_kwpack(w.float(), b.float())
            B, T, H, W = x_shape[0], x_shape[1] - rec["t_pad"], x_shape[2], x_shape[3]
            video = _grid((B, 3, T, H, W), "x", gen)
            x = self.orig["ingest_kwpack"](video.float(), rec["t_pad"], pk2)
        elif pk.epi_mode == 1 or pk.Ci_tc != pk.Ci:          # fc1 + GEGLU / fc2 of a FeedForward (pack_ff)
            C_, I = (pk.Ci, pk.Co // 2) if pk.epi_mode == 1 else (pk.Co, pk.Ci)
            w1, b1 = _grid((2 * I, C_), "w", gen), _grid(2 * I, "b", gen)
            w2, b2 = _grid((C_, I), "w", gen), _grid(C_, "b", gen)
            fc1, fc2 = pack_ff(w1.float()[..., None, None, None], b1.float(), w2.float()[..., None, None, None], b2.float(), BF)
            pk2 = fc1 if pk.epi_mode == 1 else fc2
            w, b = (w1, b1) if pk.epi_mode == 1 else (w2[..., None, None, None], b2)
            x = _grid(x_shape, "x", gen)
        else:
            w, b = _grid((pk.Co, pk.Ci, *pk.k), "w", gen), _grid(pk.Co, "b", gen)
            if pk.bias is None:           # the attention projections have no bias
                b = torch.zeros_like(b)
            b_pk = None if pk.bias is None else b.float()
            if kind == "down":
                pk2 = pack_conv(w[:, :, 0].float(), b_pk, BF)
                pack_conv_down_space(pk2, w[:, :, 0].float())
            else:
                q = {SHUFFLE_SPACE: 4, SHUFFLE_TIME: 2}.get(rec["shuffle"], 1)
                pk2 = pack_conv(w.float(), b_pk, BF, k=pk.k, shuffle_q=q)
            pk2.epi_mode = pk.epi_mode
            x = _grid(x_shape, "x", gen)
        if rec["res"]:
            res = _grid(rec["y_shape"], "x", gen)
            kw["res"] = res.to(BF).contiguous()
        os = None
        if rec.get("os"):         # a per-clip oscale on its own dyadic grid
            n, e = REPLAY_GRID["os"]
            os = torch.randint(1, n + 1, (x_shape[0], pk.Co), generator=gen, device="cuda").double() * 2.0 ** -e
            kw["oscale"] = os.float()
        kind2, y = _ran(self.eng, lambda: self.orig["conv"](x.to(BF).contiguous(), pk2, **kw))
        what = f"replay of {rec['flavour']} conv x {x_shape}"
        assert kind2 == kind, f"{what}: ran {kind2}, the recorded call ran {kind}"
        self._done(n0, what)
        rec2 = dict(rec, pk=pk2)
        self._check_conv(rec2, x, y, what, exact=True, w=w, b=b, res=res, video=video, defects=defects, os=os)
        rec.setdefault("rejected", []).extend(rec2.get("rejected", []))

    def _replay_ru(self, rec, gen, defects):
        x_shape, k = rec["x_shape"], rec["k"]
        C_ = x_shape[-1]
        p = next(v for v in self.eng._packs.values() if isinstance(v, dict) and "conv3" in v and "wk" in v
                 and v["conv3"].Co == C_)
        w3, b3 = _grid((C_, C_, *k), "w", gen), _grid(C_, "b", gen)
        w1, b1 = _grid((C_, C_, 1, 1, 1), "w", gen), _grid(C_, "b", gen)
        p2 = dict(p, conv3=pack_conv(w3.float(), b3.float(), BF), conv1=pack_conv(w1.float(), b1.float(), BF))
        x = _grid(x_shape, "x", gen)
        n0 = len(self.guard.allocs)
        kind, _ = _ran(self.eng, lambda: self.orig["residual_unit"](x.to(BF).contiguous(), p2))
        what = f"replay of the fused RU x {x_shape}"
        assert kind == "ru", f"{what}: ran {kind}"
        y = self._alloc(n0, x_shape)
        self._check_ru(rec, p2, x, y, what, exact=True, w3=w3, b3=b3, w1=w1, b1=b1, defects=defects)
        self._done(n0, what)


def _expected_calls(m):
    """Calls per kind the stages imply: conv_in and conv_out; one conv per space / time down- or up-sampler; qkv, out,
    fc1, fc2 per attention stage (q, kv, out, fc1, fc2 per linear attention stage) and its two rmsnorms; per
    ResidualUnit the fused kernel (C = 64 / 128) or two convs and squeeze_excite_residual."""
    n = dict(conv=2, ru=0, se=0, rmsnorm=0, quantize=1, codes=1)
    for st in list(m.stages) * 2:
        if st.kind == "residual":
            fused = st.dim in (64, 128)
            n["ru"] += st.count if fused else 0
            n["conv"] += 0 if fused else 2 * st.count
            n["se"] += 0 if fused else st.count
        elif st.kind in ("compress_space", "compress_time"):
            n["conv"] += 1
        elif st.kind in ("attend_space", "attend_time", "linear_attend_space"):
            n["conv"] += 5 if st.kind == "linear_attend_space" else 4
            n["rmsnorm"] += 2
        else:
            raise AssertionError(f"stage {st.kind} is not in the benchmark's configs")
    return n


def _summary(calls):
    """{flavour: (checked calls, largest total tiles, largest tiles per CTA)} of the wgmma calls."""
    out = {}
    for c in calls:
        if "plan" not in c:
            continue
        n, tot, per = out.get(c["flavour"], (0, 0, 0))
        out[c["flavour"]] = (n + 1, max(tot, c["plan"]["total"]), max(per, -(-c["plan"]["total"] // c["plan"]["grid"])))
    return out


def _replay_key(c):
    pk = c.get("pk")
    return (c["flavour"], c["x_shape"], c.get("k"), c.get("stride"), c.get("pad"), c.get("out_sp"), c.get("act"),
            c.get("shuffle"), c.get("res"), c.get("out_cf"),
            None if pk is None else (pk.Ci, pk.Co, pk.k, pk.Ci_tc, pk.Co_tc, pk.epi_mode, pk.w_down is not None))


def _defect_targets(calls):
    """The replays whose bound must reject the pipeline defects: the first fused RU of each width, the first 512- /
    1024-channel 3x3x3 EPI_PLAIN conv, conv_out."""
    want = {}
    for c in calls:
        if c.get("flavour") in ("ru_c64", "ru_c128"):
            want.setdefault(c["flavour"], id(c))
        elif c.get("flavour") == "plain" and c["pk"].Co in (512, 1024) and c["pk"].k == (3, 3, 3):
            want.setdefault("plain", id(c))
        elif c.get("flavour") == "ragged_cf":
            want.setdefault("conv_out", id(c))
    return want


@pytest.mark.parametrize("workload", ["readme", "cfg4"])
def test_bench_step_calls_vs_float64(monkeypatch, workload):
    model, clips, size = _workload(workload)
    eng = model.engine
    video = synth_data.synth_video(clips, 3, FRAMES, size, seed=1000).cuda()
    rec = _Recorder(monkeypatch, model)
    with torch.no_grad():
        codes = model.tokenize(video)
        recon = model.decode_from_code_indices(codes)
    torch.cuda.synchronize()
    _EAGER[workload] = (codes.clone(), recon.clone())
    calls = rec.calls
    # ---- structure: calls per kind, kernels, flavours ----
    got = {op: sum(c["op"] == op for c in calls) for op in ("conv", "ru", "se", "rmsnorm", "quantize", "codes")}
    want = _expected_calls(model)
    print(f"\n{workload}: calls checked per kind {got}")
    assert got == want, f"calls per kind {got}, the stages imply {want}"
    assert eng.simt_conv_calls == 0 and not any(c["kind"] == "simt" for c in calls if c["op"] in ("conv", "ru"))
    assert sum(c["kind"] == "ru" for c in calls) == eng.fused_ru_calls
    summ = _summary(calls)
    for fl, (n, tot, per) in sorted(summ.items()):
        print(f"  {fl:12s} {n:3d} calls, largest {tot:6d} tiles = {per:3d} tiles per CTA on {rec.n_sm} SMs")
    if workload == "readme":
        assert set(summ) == set(FLAVOURS), sorted(summ)
        few = {fl: per for fl, (n, tot, per) in summ.items() if not any(
            c.get("flavour") == fl and c["plan"]["total"] > 2 * c["plan"]["grid"] for c in calls if "plan" in c)}
        assert not few, f"flavours never run with more than 2 tiles per CTA: {few}"
        first_ru = next(c for c in calls if c["op"] == "ru")
        assert first_ru["plan"]["total"] == 5120, first_ru["plan"]
    # ---- exact replay of every distinct wgmma call, the pipeline defects at the named targets ----
    targets = set(_defect_targets(calls).values())
    gen = torch.Generator(device="cuda").manual_seed(7)
    seen, rejected = set(), {}
    for c in calls:
        if c["op"] not in ("conv", "ru"):
            continue
        key = _replay_key(c)
        if key in seen and id(c) not in targets:
            continue
        seen.add(key)
        rec.replay(c, gen, defects=id(c) in targets)
        if id(c) in targets:
            rejected[c["flavour"] + f" C{c['x_shape'][-1]}"] = c.get("rejected", [])
    rec._done(0, "allocations outside the checked calls")
    print(f"  {len(seen)} distinct wgmma calls replayed exactly; perturbed references rejected: {rejected}")
    names = {"one ring stage missing", "previous tile's accumulators not reset"}
    assert len(rejected) == 4, rejected
    assert all(set(v) == names for v in rejected.values()), rejected


@pytest.mark.parametrize("pdl", [False, True], ids=["pdl_off", "pdl_on"])
def test_bench_launch_mode_matches_eager(pdl):
    """The README step through StreamLanes(model, 3) with CUDA graphs (as bench.py runs it), 3 x lanes steps on distinct
    batches, equal bit for bit to the eager step of each batch; batch 0's eager step is the one the float64 test checked."""
    model, clips, size = _workload("readme")
    lanes_n = 3
    batches = [synth_data.synth_video(clips, 3, FRAMES, size, seed=1000 + i).cuda() for i in range(3 * lanes_n)]

    def step(v):
        codes = model.tokenize(v)
        return codes, model.decode_from_code_indices(codes)

    with torch.no_grad():
        want = [tuple(t.clone() for t in step(v)) for v in batches]
    if "readme" in _EAGER:
        assert torch.equal(want[0][0], _EAGER["readme"][0]) and torch.equal(want[0][1], _EAGER["readme"][1])
    model.cuda_graphs = True
    model.pdl = pdl
    lanes = StreamLanes(model, lanes_n)
    got = []
    for v in batches:                 # every lane: plain call, capture, replay; copied before the lane's next replay
        res, _ = lanes.run(lambda v_: tuple(t.clone() for t in step(v_)), v)
        got.append(res)
    lanes.join()
    torch.cuda.synchronize()
    for i, ((gc, gv), (wc, wv)) in enumerate(zip(got, want)):
        assert torch.equal(gc, wc), f"step {i} (lane {i % lanes_n}): codes differ from the eager step"
        assert torch.equal(gv, wv), f"step {i} (lane {i % lanes_n}): reconstruction differs from the eager step"
    assert len({k[3] for k in model._graphs}) == lanes_n
