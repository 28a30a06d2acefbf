"""Every kernel call of tokenize + decode_from_code_indices under each non-default constructor option, checked one call at
a time against float64 at the README widths (image_size 128, init_dim 64, max_dim 512).  The README constructor is
tests/test_bench_calls_gpu.py's; the mini_* goldens check these options only at 32^2 / 16..64 channels, where the bf16
convs mostly take other kernels and the end-to-end budgets would hide a per-call slip.

Configs (OPTION_CONFIGS; tests/test_option_calls_cpu.py pins their kernels, call counts and slab plans without a GPU):
  fsq (bench.WORKLOADS["fsq"]), cond_deep / cond_wide (Conv3DMod at 512 / 64 channels, a distinct cond per clip), gateloop
  (the scan at 64^2 pixels, 128 / 256 channels), sff (separate_first_frame_encoding), pad_reflect / pad_replicate /
  pad_circular, mc_spherical (two spherical LFQ codebooks), noff (video_contains_first_frame=False).

Part 1, real data.  tests/test_bench_calls_gpu.py's recorder (NaN-filled, sentinel-bordered allocations, per-clip float64
references, the kernel tests' bounds), extended by _OptionRecorder:
  * Engine.conv with oscale: forward64 with the clip's own oscale row;
  * the CUDA-core conv only for the calls named in SIMT_ROLES (the 3-channel conv_in under a pad mode and sff's two
    conv_in parts); every other bf16 call on a wgmma kernel;
  * residual_unit_mod: dense_small (to_cond and the cond stems) against float64 act(x W^T + b), mod_prepare's scale_in /
    inv_norm from the kernel's own fp32 inputs, scale_channels within one rounding, both convs as above;
  * gateloop: the scan against the float64 recurrence of the call's own bf16 qkva and x (test_simt_ops_gpu.gateloop64);
  * causal_conv_padded: the padded input equal to F.pad(x, mode) bit for bit, then the conv with pad (0, 0, 0);
  * sff: each part's input equal to its frames of the clip, and conv_in's feature map / conv_out's reconstruction equal
    to the parts placed at their frames (zero time-padding frames), bit for bit;
  * FSQ: indices exact except where the float64 bounded value lies within its allowance of a rounding point (test_fsq's
    bound, fsq64), the decode against fsq_indices_to_codes; spherical LFQ also its per-codebook normalised pre-sign values.
Negative controls (each must be rejected): clip 0's oscale used for another clip, the gateloop output taken from the
state before the update, reflect padding that includes the edge pixel, sff's first frame read from frame tp + 1, FSQ
indices with the mixed-radix digits reversed.  (The Conv3DMod conv has no bias, so "oscale applied after the bias" is the
same arithmetic there; tests/test_conv_forward_gpu.py rejects it on biased oscale convs.)

Part 2, exact replay: every distinct wgmma call again on REPLAY_GRID operands, oscale on its {1..8} / 2^3 grid (so only
the oscale product and the bias add round).  At the 512-channel Conv3DMod of cond_deep, the 64-channel one of cond_wide
and the first qkva conv of gateloop the bound must reject one ring stage missing and the previous tile's accumulators
not reset at the schedule's last tile.  The pad-0 conv_out runs on the tap-wise kernel over a plane two rows and columns
larger than its output and is replayed exactly.

Part 3, streaming: cond_wide, gateloop and sff through tokenize_stream / decode_stream with tests/test_stream_gpu.py's
chunk schedules equal the whole-clip codes and reconstruction bit for bit; the streamed Conv3DMod ran on the slab kernel
with history frames."""
import math

import pytest
import torch
import torch.nn.functional as F

import synth_data
from oracle import restated as R
from tests.test_bench_calls_gpu import _Recorder, _replay_key, _summary
from tests.test_conv_forward_gpu import _ran, forward64
from tests.test_option_calls_cpu import (OPTION_CONFIGS, SIMT_ROLES, expected_option_calls, option_kw, tap_boxes)
from tests.test_simt_ops_gpu import (U, _check, _proj_err, _quant_sd, _rejects, dense_small64, fsq64, gateloop64,
                                     lfq_presign64, mod_prepare64, scale_channels64)
from tests.test_stream_gpu import _decode_stream, _schedules, _tokenize_stream

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_NONE

pytestmark = pytest.mark.gpu

BF, F64 = torch.bfloat16, torch.float64
_WHOLE = {}          # config -> (codes, reconstruction) of part 1, for the streaming test


def _model(name):
    torch.manual_seed(0)
    model = VideoTokenizer(**option_kw(name))
    synth_data.fill_state_dict_(model, 0)
    return model.cuda().bfloat16().eval()


def _inputs(name, model):
    cfg = OPTION_CONFIGS[name]
    video = synth_data.synth_video(cfg["clips"], 3, cfg["frames"], 128, seed=1000).cuda()
    cond = None
    if model.has_cond:            # a distinct cond per clip: a per-clip oscale read from the wrong clip differs
        g = torch.Generator(device="cuda").manual_seed(3)
        cond = torch.randn((cfg["clips"], model.dim_cond), generator=g, device="cuda").to(BF)
    return video, cond, cfg.get("ff", True)


def _run(model, video, cond, ff):
    with torch.no_grad():
        if cond is None and ff:
            codes = model.tokenize(video)
        else:
            codes = model(video, cond=cond, return_codes=True, video_contains_first_frame=ff)
        recon = model.decode_from_code_indices(codes, cond=cond, video_contains_first_frame=ff)
    torch.cuda.synchronize()
    return codes, recon


class _OptionRecorder(_Recorder):
    """The benchmark test's recorder plus the entry points of the non-default options (module docstring)."""

    EXTRA = ("dense_small", "residual_unit_mod", "gateloop", "causal_conv_padded", "conv_in", "conv_out")

    def __init__(self, monkeypatch, model):
        super().__init__(monkeypatch, model)
        self.orig.update({k: getattr(self.eng, k) for k in self.EXTRA})
        for k in self.EXTRA:
            monkeypatch.setattr(self.eng, k, getattr(self, k))
        self.log = None           # (role, x, y) of every conv while conv_in / conv_out run
        self.pad_inputs = []
        self.last_dense = None
        self.controls = {}
        P = self.eng._packs
        self.roles = {id(P["conv_in"]): "conv_in", id(P["conv_out"]): "conv_out"}
        for k in ("conv_in_ff", "conv_out_ff"):
            if k in P:
                self.roles[id(P[k])] = k.replace("_ff", "_first_frame")
        for k, v in P.items():
            if isinstance(v, dict) and "qkva" in v:
                self.roles[id(v["qkva"])] = "qkva"
            if isinstance(v, dict) and "S" in v:
                self.roles[id(v["conv3"])], self.roles[id(v["conv1"])] = "mod_conv3", "mod_conv1"

    def _control(self, name, what, rejected):
        assert rejected, f"{what}: the check does not reject {name}"
        self.controls.setdefault(name, what)

    # ---------------------------------------------------------------- Engine.conv
    def _conv_record(self, x, pk, kw, y, kind):
        d = super()._conv_record(x, pk, kw, y, kind)
        d["role"] = self.roles.get(id(pk), "other")
        d["simt_ok"] = d["role"] in SIMT_ROLES
        if kind == "slab" and d["os"]:
            d["flavour"] = "oscale"
        elif kind == "slab" and d["role"] == "qkva":
            d["flavour"] = "qkva"
        return d

    def conv(self, x, pk, **kw):
        y = super().conv(x, pk, **kw)
        if self.log is not None:
            self.log.append((self.calls[-1]["role"], x, y))
        return y

    def _check_conv(self, rec, x, y, what, exact=False, w=None, b=None, res=None, video=None, defects=False, os=None):
        super()._check_conv(rec, x, y, what, exact=exact, w=w, b=b, res=res, video=video, defects=defects, os=os)
        control = "clip 0's oscale (inv_norm) used for another clip"
        if os is not None and not exact and x.shape[0] > 1 and control not in self.controls:
            xs, w_, b_, kw = self._conv_ref_args(rec, x)
            i = x.shape[0] - 1
            _, acc = forward64(xs(i), w_, b_, os[i:i + 1].double(), None, dtype=BF, **kw)
            wrong, _ = forward64(xs(i), w_, b_, os[:1].double(), None, dtype=BF, **kw)
            self._control(control, what, _excess_gt0(y[i:i + 1], wrong, acc))

    # ---------------------------------------------------------------- conditioning
    def dense_small(self, x, w, b, act=ACT_NONE):
        n0 = len(self.guard.allocs)
        y = self.orig["dense_small"](x, w, b, act)
        what = f"call {len(self.calls)}: dense_small {tuple(x.shape)} x {tuple(w.shape)}"
        self._done(n0, what)
        ref, acc, _ = dense_small64(x.double(), w.double(), None if b is None else b.double(), act)
        _check(y, ref, torch.float32, acc, what)
        self.last_dense = y
        self.calls.append(dict(op="dense", kind="simt"))
        return y

    def residual_unit_mod(self, x, p, cond_e, ss=None):
        assert ss is None
        n0 = len(self.guard.allocs)
        out = self.orig["residual_unit_mod"](x, p, cond_e)
        what = f"call {len(self.calls)}: residual_unit_mod {tuple(x.shape)}"
        B, T, H, W, C_ = x.shape
        torch.cuda.synchronize()
        # allocations left after the checked dense_small / conv calls released theirs: scale_in, inv_norm, the scaled x
        scale_in, inv_norm = self._alloc(n0, (B, C_)), self._alloc(n0 + 1, (B, C_))
        xs = self._alloc(n0 + 2, x.shape)
        si_ref, inv_ref, acc, _ = mod_prepare64(self.last_dense.double(), p["S"].double(), p["eps"])
        _check(scale_in, si_ref, torch.float32, 0.0, f"{what}: mod_prepare scale_in")
        _check(inv_norm, inv_ref, torch.float32, acc, f"{what}: mod_prepare inv_norm")
        ref, acc = scale_channels64(x.double().reshape(B, -1, C_), scale_in.double(), BF)
        _check(xs.reshape(B, -1, C_), ref, BF, acc, f"{what}: scale_channels")
        self._done(n0, what)
        self.calls.append(dict(op="mod", kind="simt"))
        return out

    # ---------------------------------------------------------------- gateloop
    def gateloop(self, x, p, ss=None):
        assert ss is None
        n0 = len(self.guard.allocs)
        log, self.log = self.log, []
        out = self.orig["gateloop"](x, p)
        (_, _, qkva), self.log = self.log[-1], log
        what = f"call {len(self.calls)}: gateloop scan {tuple(x.shape)}"
        self._done(n0, what)
        B, T, H, W, C_ = x.shape
        ref, acc, wrong = gateloop64(qkva.double().reshape(B, T, H * W, 3 * C_), x.double().reshape(B, T, H * W, C_))
        got = out.reshape(B, T, H * W, C_)
        _check(got, ref, BF, acc, what)
        self._control("the gateloop output taken from the state before the update", what, _excess_gt0(got, wrong, acc))
        del ref, acc, wrong
        self.calls.append(dict(op="gateloop", kind="simt", P=H * W, C=C_))
        return out

    # ---------------------------------------------------------------- padding modes
    def causal_conv_padded(self, x, pk, pad_mode):
        n0 = len(self.guard.allocs)
        y = self.orig["causal_conv_padded"](x, pk, pad_mode)
        B, T, H, W, C_ = x.shape
        kt, kh, kw = pk.k
        what = f"call {len(self.calls)}: mv2_pad_cl {pad_mode} {tuple(x.shape)}"
        if pad_mode != "constant" and kt - 1 < T:
            torch.cuda.synchronize()
            xp = self._alloc(n0, (B, T + kt - 1, H + 2 * (kh // 2), W + 2 * (kw // 2), C_))
            pads = (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0)

            def pad(mode):
                return F.pad(x.float().permute(0, 4, 1, 2, 3), pads, mode=mode).permute(0, 2, 3, 4, 1).to(x.dtype)
            assert torch.equal(xp, pad(pad_mode)), f"{what}: differs from F.pad(x, mode={pad_mode!r})"
            if pad_mode == "reflect":
                self._control("reflect padding that includes the edge pixel", what, not torch.equal(xp, pad("replicate")))
            self.pad_inputs.append(x)
            self.calls.append(dict(op="pad", kind="simt", mode=pad_mode))
        self._done(n0, what)
        return y

    # ---------------------------------------------------------------- conv_in / conv_out assembly
    def conv_in(self, video, first_frame=True, ss=None, sff_rest=False):
        assert ss is None and not sff_rest
        m = self.m
        self.log, self.pad_inputs = [], []
        x = self.orig["conv_in"](video, first_frame)
        log, self.log = self.log, None
        t_pad = m.time_padding if first_frame else 0
        v = video.to(BF).permute(0, 2, 3, 4, 1)
        what = f"conv_in {tuple(video.shape)}"
        if m.separate_first_frame_encoding and first_frame:
            (r0, x0, y0), (r1, x1, y1) = log
            assert (r0, r1) == ("conv_in_first_frame", "conv_in"), (r0, r1)
            assert torch.equal(x0, v[:, :1]) and torch.equal(x1, v[:, 1:]), f"{what}: a part's input frames"
            zeros = torch.zeros_like(x[:, :t_pad])
            assert torch.equal(x, torch.cat((zeros, y0, y1), 1)), f"{what}: the feature map is not [0 x tp, first, rest]"
        elif m.conv_in.pad_mode != "constant":
            assert len(self.pad_inputs) == 1 and len(log) == 1 and log[0][2] is x
            assert torch.equal(self.pad_inputs[0], F.pad(v, (0, 0, 0, 0, 0, 0, t_pad, 0))), f"{what}: the padded conv's input"
        return x

    def conv_out(self, x, first_frame=True, ss=None, sff_rest=False):
        assert ss is None and not sff_rest
        m = self.m
        self.log, self.pad_inputs = [], []
        recon = self.orig["conv_out"](x, first_frame)
        log, self.log = self.log, None
        tp = m.time_padding if first_frame else 0
        what = f"conv_out {tuple(x.shape)}"
        torch.cuda.synchronize()
        if m.separate_first_frame_encoding and first_frame:
            (r0, x0, y0), (r1, x1, y1) = log
            assert (r0, r1) == ("conv_out_first_frame", "conv_out"), (r0, r1)
            assert torch.equal(x0, x[:, tp:tp + 1]) and torch.equal(x1, x[:, tp + 1:]), f"{what}: a part's input frames"
            assert torch.equal(recon, torch.cat((y0, y1), 1).permute(0, 4, 1, 2, 3)), f"{what}: the assembled frames"
            self._control("sff's first frame read from frame tp + 1", what, not torch.equal(x0, x[:, tp + 1:tp + 2]))
        elif m.conv_out.pad_mode != "constant":
            (r, _, y), = log
            assert self.pad_inputs == [x] and r == "conv_out"
            assert torch.equal(recon, y[:, tp:].permute(0, 4, 1, 2, 3)), f"{what}: the channels-first copy"
        else:
            assert len(log) == 1 and log[0][2] is recon        # the channels-first conv_out: checked as a conv call
        return recon

    # ---------------------------------------------------------------- quantisers
    def _qprm(self):
        P = self.eng._packs["quant"]
        return {k: P[k].double() for k in ("win", "bin", "wout", "bout")}

    def quantize_cl(self, x, want_quantized=True, want_aux=False):
        qz = self.m.quantizers
        if not self.m.use_fsq:
            q, idx, aux = super().quantize_cl(x, want_quantized, want_aux)
            if qz.spherical:
                self._spherical_presign(x, idx)
            return q, idx, aux
        n0 = len(self.guard.allocs)
        q, idx, aux = self.orig["quantize_cl"](x, want_quantized, want_aux)
        what = f"call {len(self.calls)}: quantize_cl (FSQ) {tuple(x.shape)}"
        self._done(n0, what)
        nc, C_ = qz.num_codebooks, x.shape[-1]
        N = x[..., 0].numel()
        prm = self._qprm()
        f = fsq64(x.double().reshape(N, C_), prm, list(qz.levels), nc)
        amb = f["ambiguous"]
        assert amb.sum().item() <= max(2, N // 100), f"{what}: {amb.sum().item()} ambiguous digits"
        got = idx.reshape(N, nc).long()
        assert torch.equal(got[~amb], f["idx"].long()[~amb]), what
        self._control("FSQ indices with the mixed-radix digits reversed", what,
                      (got != f["reversed"].long()).sum().item() > amb.sum().item())
        if q is not None:
            ok = ~amb.any(dim=1)
            _check(q.reshape(N, C_)[ok], f["q"][ok], BF, f["acc_q"].expand(N, C_)[ok], f"{what}: quantized")
        if aux is not None:
            _check(aux, f["bounded"], torch.float32, f["err"], f"{what}: bounded values")
        self.calls.append(dict(op="quantize", kind="simt", ambiguous=amb.sum().item(), N=N))
        return q, idx, aux

    def _spherical_presign(self, x, idx):
        """The pre-sign values of the same call (want_aux): the fp32 projection, per codebook L2-normalised."""
        qz = self.m.quantizers
        n0 = len(self.guard.allocs)
        _, idx2, aux = self.orig["quantize_cl"](x, False, True)
        what = f"call {len(self.calls) - 1}: quantize_cl pre-sign values (spherical, {qz.num_codebooks} codebooks)"
        self._done(n0, what)
        assert torch.equal(idx2, idx), what
        prm = self._qprm()
        N, C_ = x[..., 0].numel(), x.shape[-1]
        x64 = x.double().reshape(N, C_)
        clamp = qz.soft_clamp_input_value
        lin = x64 @ prm["win"].T + prm["bin"]
        p64 = torch.tanh(lin / clamp) * clamp if clamp else lin
        err = _proj_err(x64, prm) + 4 * U * p64.abs()
        ref, acc = lfq_presign64(p64, err, qz.num_codebooks, qz.codebook_dim, True)
        _check(aux, ref, torch.float32, acc, what)
        self.calls[-1]["presign"] = True

    def codes_to_quantized_cl(self, codes):
        if not self.m.use_fsq:
            return super().codes_to_quantized_cl(codes)
        n0 = len(self.guard.allocs)
        q = self.orig["codes_to_quantized_cl"](codes)
        what = f"call {len(self.calls)}: codes_to_quantized_cl (FSQ) {tuple(codes.shape)}"
        self._done(n0, what)
        qz, prm = self.m.quantizers, self._qprm()
        levels, nc, C_ = list(qz.levels), qz.num_codebooks, q.shape[-1]
        N = math.prod(codes.shape[:4])
        sd = {k: v.cpu() for k, v in _quant_sd(prm, len(levels)).items()}
        c = codes.reshape(N, nc) if nc > 1 else codes.reshape(N)
        want = R.fsq_indices_to_codes(c.cpu(), sd, levels, F64, nc).cuda()
        acc = (len(levels) * nc + 2) * U * (prm["wout"].abs().sum(dim=1) + prm["bout"].abs())
        _check(q.reshape(N, C_), want.reshape(N, C_), BF, acc.expand(N, C_), what)
        self.calls.append(dict(op="codes", kind="simt"))
        return q


def _excess_gt0(out, wrong, acc):
    """True when the bound rejects the perturbed reference `wrong`."""
    try:
        _rejects(out, wrong, BF, acc, "")
        return True
    except AssertionError:
        return False


def _defect_targets(name, calls):
    """The replays whose bound must reject the pipeline defects: the Conv3DMod (oscale) conv of cond_deep (512 channels)
    and cond_wide (64 channels), the first qkva conv of gateloop."""
    for c in calls:
        if name in ("cond_deep", "cond_wide") and c.get("flavour") == "oscale" and \
                c["pk"].Co == {"cond_deep": 512, "cond_wide": 64}[name]:
            return {id(c): f"Conv3DMod C{c['pk'].Co}"}
        if name == "gateloop" and c.get("flavour") == "qkva":
            return {id(c): f"qkva C{c['pk'].Ci}"}
    return {}


@pytest.mark.parametrize("name", list(OPTION_CONFIGS))
def test_option_calls_vs_float64(monkeypatch, name):
    model = _model(name)
    eng = model.engine
    video, cond, ff = _inputs(name, model)
    model.engine.prepare()
    rec = _OptionRecorder(monkeypatch, model)
    torch.cuda.reset_peak_memory_stats()
    codes, recon = _run(model, video, cond, ff)
    _WHOLE[name] = (codes.clone(), recon.clone())
    calls = rec.calls
    # ---- structure: calls per kind, the CUDA-core calls by name, flavours and tiles per CTA ----
    ops = ("conv", "ru", "se", "rmsnorm", "quantize", "codes", "dense", "mod", "gateloop", "pad")
    got = {op: sum(c["op"] == op for c in calls) for op in ops}
    want = expected_option_calls(model, ff)
    print(f"\n{name}: calls checked per kind {got}")
    assert got == want, f"calls per kind {got}, the stages imply {want}"
    simt = [c["role"] for c in calls if c["op"] == "conv" and c["kind"] == "simt"]
    assert simt == OPTION_CONFIGS[name].get("simt", []), f"calls on the CUDA-core conv: {simt}"
    assert eng.simt_conv_calls == len(simt)
    kinds = sorted({(c["role"], c["kind"]) for c in calls if c["op"] == "conv" and c["role"] != "other"})
    print(f"  kernels of the option-specific calls: {kinds}")
    summ = _summary(calls)
    for fl, (n, tot, per) in sorted(summ.items()):
        print(f"  {fl:12s} {n:3d} calls, largest {tot:6d} tiles = {per:3d} tiles per CTA on {rec.n_sm} SMs")
    many = {fl for fl in ("oscale", "qkva") if any(c.get("flavour") == fl and c["plan"]["total"] > 2 * c["plan"]["grid"]
                                                  for c in calls if "plan" in c)}
    assert many >= set(OPTION_CONFIGS[name].get("many_tiles", ())), (many, summ)
    if name.startswith("pad_"):
        tap = [c for c in calls if c["op"] == "conv" and c["role"] == "conv_out"]
        assert len(tap) == 1 and tap[0]["kind"] == "tap" and tap[0]["pad"] == (0, 0, 0), tap
        _, _, Hi, Wi, _ = tap[0]["x_shape"]
        _, Ho, Wo = tap[0]["out_sp"]
        bw, bh, bt = tap_boxes(Ho, Wo)
        print(f"  pad-0 conv_out on the tap-wise kernel: input plane {Hi}x{Wi}, output {Ho}x{Wo}, box {bw}x{bh}x{bt}: "
              f"{-(-Ho // bh)} boxes along H, {-(-Wo // bw)} along W")
        assert (Hi, Wi) == (Ho + 2, Wo + 2) and -(-Ho // bh) > 1
    print(f"  negative controls rejected: {sorted(rec.controls)}")
    assert set(rec.controls) >= set(OPTION_CONFIGS[name].get("controls", ())), rec.controls
    # ---- exact replay of every distinct wgmma call, the pipeline defects at the named targets ----
    targets = _defect_targets(name, calls)
    gen = torch.Generator(device="cuda").manual_seed(7)
    seen, rejected = set(), {}
    for c in calls:
        if c["op"] not in ("conv", "ru") or c["kind"] == "simt":
            continue
        key = _replay_key(c)
        if key in seen and id(c) not in targets:
            continue
        seen.add(key)
        rec.replay(c, gen, defects=id(c) in targets)
        if id(c) in targets:
            rejected[targets[id(c)]] = c.get("rejected", [])
    rec._done(0, "allocations outside the checked calls")
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"  {len(seen)} distinct wgmma calls replayed exactly; defects rejected: {rejected}; peak {peak:.1f} GiB")
    names = {"one ring stage missing", "previous tile's accumulators not reset"}
    if name in ("cond_deep", "cond_wide", "gateloop"):
        assert len(rejected) == 1 and all(set(v) == names for v in rejected.values()), rejected


STREAM_CONFIGS = ["cond_wide", "gateloop", "sff"]


@pytest.mark.parametrize("name", STREAM_CONFIGS)
def test_option_stream_equals_whole_clip(monkeypatch, name):
    """The same clips pushed in chunks (tests/test_stream_gpu.py's schedules) give the whole-clip codes and reconstruction
    bit for bit; the whole-clip outputs are the ones part 1 checked."""
    model = _model(name)
    eng = model.engine
    video, cond, ff = _inputs(name, model)
    codes, recon = _run(model, video, cond, ff)
    if name in _WHOLE:
        assert torch.equal(codes, _WHOLE[name][0]) and torch.equal(recon, _WHOLE[name][1])
    seen = []
    orig = eng.conv

    def conv(x, pk, **kw):        # which kernel each streamed conv ran, and whether it read history frames
        ss = kw.get("ss")
        hist = ss is not None and ss.get("hist") is not None
        kind, y = _ran(eng, lambda: orig(x, pk, **kw))
        seen.append((kw.get("oscale") is not None, hist, kind))
        return y
    monkeypatch.setattr(eng, "conv", conv)
    monkeypatch.setattr(eng, "conv_log", [])
    tdf = model.time_downsample_factor
    n_lat = codes.shape[1]
    scheds = _schedules(tdf, n_lat, ff)
    assert any(tdf in s[1:] for s in scheds), scheds            # a push of one latent frame after the first
    with torch.no_grad():
        for sched in scheds:
            assert torch.equal(_tokenize_stream(model, video, sched, cond, ff), codes), sched
        for sizes in ([n_lat], [1] * n_lat, [1, 2] + [1] * (n_lat - 3)):
            got = _decode_stream(model, codes, sizes, cond, ff)
            assert torch.equal(got, recon), sizes
    torch.cuda.synchronize()
    if model.has_cond:
        assert any(os and hist and kind == "slab" for os, hist, kind in seen), "no streamed Conv3DMod on the slab with history"
    print(f"\n{name}: {len(scheds)} encoder and 3 decoder schedules equal the whole-clip outputs; "
          f"{sum(h for _, h, _ in seen)} conv calls read history frames")
