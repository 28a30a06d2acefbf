"""Every kernel call the README training step makes on the GAN discriminator (gan.py) and the VGG perceptual loss (vgg.py),
at the trainer's own shapes, checked one call at a time against float64.

The workload is the one of tools/perceptual_step_time.py: VideoTokenizer(image_size=128, init_dim=64, max_dim=512,
codebook_size=1024, layers=README_LAYERS, vgg=build_vgg(VGG16_CFG, 4096)), synth_data weights, bf16, train() with the
VGG in eval() (its classifier dropout is a torch multiply, not a kernel under test), 4 clips of 3 x 17 x 128 x 128.  After
one warm-up step (so that the discriminator's and the VGG's packs and engines exist) it runs a generator step (the
discriminator forward and backward with the image gradient, the VGG on the real and the reconstructed frames, the VGG's
data gradient) and a discriminator step (two discriminator forwards and backwards, no gradient penalty).  The
discriminator's widths are 3 -> 512 -> 512 ... 512 (its `dim` is the tokenizer's last stage width), six blocks, last map
4 x 4.  The tokenizer's own engine is checked by tests/test_train_tokenizer_calls_gpu.py.

Part 1, real data.  The entry points of the discriminator's and the VGG's engine instances (conv, ingest_kwpack, rmsnorm,
maxpool2x2, maxpool2x2_backward, mse) and the runners' TapeRunner._dgrad / DiscrRunner._dgrad_s2 are wrapped; each call
is checked when it returns (synchronise, float64 reference from the call's own bf16 operands one image at a time, check,
free).  Every output starts NaN-filled between two sentinels (_Guard).  References and bounds are the kernel tests':
  * Engine.conv: forward64 / geglu64 (tests/test_conv_forward_gpu.py) with the weights of pk.w, the CUDA-core layout.
    The kw-packed first convs take the module's 3x3 weights applied to the images; the unshuffle conv takes the module's
    1x1 weights applied to F.pixel_unshuffle of its input (so unshuffle_conv_weight is checked).  The two Linears that
    run as map-covering convs are checked against the module, not the pack: to_logits as F.linear of the float64 (c h w)
    flatten; the VGG's first Linear as F.adaptive_avg_pool2d to 7 x 7, flatten, F.linear.  Its pack folds the pool into
    the weights in fp32 and rounds them to bf16: each folded weight is then within (2^-8 + 2^-23) |w_fold| of the float64
    fold (bf16 rounding 2^-8 relative, the fp32 rounding before it 2^-24, their product below 2^-32), and |w_fold| <=
    the fold of |W| (the pool matrices are non-negative), so FOLD * (pool(|h|) @ |W|) is added to the bound, and the
    accumulation allowance uses (1 + 2^-7) times that sum for the rounded weights;
  * the VGG's transposed Linears (their data gradients): the float64 product with the Linear's weight; for the first
    Linear the adjoint of the average pool, as the channels-last (h, w, c) map gradient, with the fold allowance;
  * data gradients: _dgrad64 / _s2_grad64 (tests/test_conv_grad_gpu.py), float64 autograd of the forward the engine runs,
    the stride-2 ones from the module's weight (so unshuffle_dgrad_weight / stride2_1x1_dgrad_weight are checked);
  * maxpool2x2 and its backward: exactly equal to F.max_pool2d and to the gradient sent to each window's first maximum,
    masked by the ReLU; rmsnorm: _rms_ref; mse: the bound of test_mse; ingest_kwpack: exactly equal.
The linear attention kernel is checked at these lengths by tests/test_attention_gpu.py and is left out; its q, kv and out
convs and the feed-forward convs are checked as convs.  The test asserts the number of calls of each kind the module
structure implies (tests/test_train_calls_cpu.py), that each call ran the kernel of that file's table (only block 0's
conv_res and its stride-2 data gradient on the CUDA cores), and from mv2_tc_slab_plan with the device's SM count that
the 128^2 slab calls ran more than one tile on some CTAs (the 512-channel ones more than two per CTA).

Part 2, exact replay.  At depth 8192 the fp32 allowance of real data is as large as one 64-channel K chunk's share, so
every distinct wgmma call is replayed with the same entry point, shapes, arguments and packer on REPLAY_GRID operands:
every product is a multiple of 2^-8 of size <= 0.25, every partial sum up to depth 8192 is <= 2^11 and exact in fp32,
and the allowance is the epilogue's alone.  On every replayed tap call the bound must reject one missing 64-channel K
chunk; on every replayed slab conv and dgrad the ring stage of the schedule's last tile missing, and, where the CTA of
that tile ran an earlier one, that tile's accumulators not reset (_defect_deltas of tests/test_bench_calls_gpu.py).

Negative controls: LeakyReLU slope 0.2, the 2^-0.5 scale on one branch only, the logits weight read in (h w c) order,
the average-pool windows shifted by one, the depth-to-space phases swapped, and a maxpool tie sending its gradient to
the last maximum must each be rejected."""
import ctypes as C
import math
import time

import pytest
import torch
import torch.nn.functional as F

import synth_data
from tests.test_bench_calls_gpu import (_acc64, _defect_deltas, _grid, _lib_plan, _n_sm, _region,
                                        last_cta)
from tests.test_conv_forward_gpu import HEAD, _conv64, _Guard, _ran, forward64, geglu64
from tests.test_conv_grad_gpu import C_OF, _dgrad64, _gamma, _s2_grad64
from tests.test_simt_ops_gpu import U, _check, _rejects, _rms_ref
from tests.test_train_calls_cpu import CLIPS, README_TRAIN_KW, SIMT_BY_DESIGN, readme_table, step_counts

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_LEAKY_RELU, ACT_NONE, SHUFFLE_NONE
from magvit2_pytorch_b200.engine import pack_conv, pack_conv_in_kwpack, pack_ff
from magvit2_pytorch_b200.gan import (DiscrRunner, stride2_1x1_dgrad_weight, unshuffle_conv_weight,
                                      unshuffle_dgrad_weight)
from magvit2_pytorch_b200.train import TapeRunner
from magvit2_pytorch_b200.vgg import adaptive_pool_matrix

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FOLD = 2.0 ** -8 + 2.0 ** -23          # fold-and-round error of the VGG's first Linear, relative to |w_fold| (docstring)
KW_K = 3 * 32                          # GEMM depth of the kw-packed 3x3 first convs: 3 row taps x 32 packed channels


def _model():
    torch.manual_seed(0)
    m = VideoTokenizer(**README_TRAIN_KW, vgg=synth_data.build_vgg(synth_data.VGG16_CFG, 4096))
    synth_data.fill_state_dict_(m)
    synth_data.fill_discr_(m)
    synth_data.fill_vgg_(m.vgg)
    m = m.cuda().bfloat16().train()
    m.vgg.eval()
    return m


def _cf(x):
    """(B, 1, H, W, C) channels-last -> (B, C, H, W) float64."""
    return x[:, 0].double().permute(0, 3, 1, 2)


def _pool_windows(x):
    """(B, 1, H, W, C) -> (B, H/2, W/2, C, 4) float64: each 2 x 2 window in row-major order."""
    B, _, H, W, C_ = x.shape
    return x[:, 0].double().reshape(B, H // 2, 2, W // 2, 2, C_).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C_, 4)


def _pool_grad64(g, x, last=False):
    """Gradient wrt the pool's input: each window's gradient to its first (last: its last) maximum, masked by x > 0."""
    B, _, H, W, C_ = x.shape
    xw = _pool_windows(x)
    idx = 3 - xw.flip(-1).argmax(-1) if last else xw.argmax(-1)
    gw = torch.zeros_like(xw).scatter_(-1, idx[..., None], g[:, 0].double()[..., None])
    gx = gw.reshape(B, H // 2, W // 2, C_, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, C_)
    return (gx * (x[:, 0].double() > 0))[:, None]


def _pool_adjoint(gp, fmap, out_size):
    """Adjoint of adaptive_avg_pool2d (B, C, oh, ow) -> (B, C, h, w)."""
    ah, aw = (adaptive_pool_matrix(n, o).to(gp.device) for n, o in zip(fmap, out_size))
    return torch.einsum("bcyx,yh,xw->bchw", gp, ah, aw)


class _Recorder:
    """Wraps the entry points of the discriminator's and the VGG's engines; every call is checked when it returns."""

    def __init__(self, monkeypatch, m):
        self.m, self.d, self.vgg = m, m.discr, m.vgg
        engs = {"discr": m.discr._pack_cache.engine, "vgg": m._vgg_cache.engine}
        self.net = {id(e): n for n, e in engs.items()}
        self.guard = {id(e): _Guard(e) for e in engs.values()}
        self.lib, self.n_sm = engs["discr"].lib, _n_sm()
        self.simt0 = {id(e): e.simt_conv_calls for e in engs.values()}      # the warm-up's CUDA-core convs
        _, self.table = readme_table()
        self.calls, self.ingest, self.nested, self.controls = [], {}, None, {}
        self.orig = {}
        for e in engs.values():
            monkeypatch.setattr(e, "_new", self.guard[id(e)].new)
            monkeypatch.setattr(e, "conv_log", [])
            for k in ("conv", "ingest_kwpack", "rmsnorm", "maxpool2x2", "maxpool2x2_backward", "mse"):
                self.orig[(id(e), k)] = getattr(e, k)
                monkeypatch.setattr(e, k, self._bind(getattr(self, k), e))
        self.orig_dgrad, self.orig_s2 = TapeRunner._dgrad, DiscrRunner._dgrad_s2
        monkeypatch.setattr(TapeRunner, "_dgrad", self._dgrad_wrapper(TapeRunner._dgrad, "dgrad"))
        monkeypatch.setattr(DiscrRunner, "_dgrad_s2", self._dgrad_wrapper(DiscrRunner._dgrad_s2, "dgrad_s2"))
        # the packs of the forward convs -> (net, role) of the table
        P, logits = self.d._pack_cache.packs
        self.roles = {id(logits["conv"]): "logits_conv", id(logits["lin"]): "logits_lin"}
        for e in P:
            for k, role in (("net0_kw", "net0_kw"), ("net0", "net0"), ("net2", "net2"), ("down", "down")):
                if k in e:
                    self.roles[id(e[k])] = role
            self.roles[id(e["res"])] = "res" if e["res"].epi_mode == 0 else "res_scaled"
            for k in ("q", "kv", "out"):
                self.roles[id(e["attn"][k])] = k
            for k in ("fc1", "fc2"):
                self.roles[id(e["ff"][k])] = k
        vp = m._vgg_cache.packs
        for i, e in enumerate(vp["feats"]):
            self.roles[id(e["pk"])] = "conv"
            if "kw" in e:
                self.roles[id(e["kw"])] = "conv_kw"
        for j, op in enumerate(o for o in vp["ops"] if o["kind"] == "linear"):
            self.roles[id(op["pk"])], self.roles[id(op["pk_t"])] = f"linear{j + 1}", f"linear{j + 1}_t"

    @staticmethod
    def _bind(fn, eng):
        return lambda *a, **k: fn(eng, *a, **k)

    # ---------------------------------------------------------------- allocations
    def _done(self, eng, n0, what):
        """The borders of eng's allocations made since n0 unchanged; then they are no longer tracked."""
        torch.cuda.synchronize()
        allocs = self.guard[id(eng)].allocs
        for i, (buf, n, head, tail) in enumerate(allocs[n0:]):
            assert torch.equal(buf[:HEAD], head), f"{what}: store before allocation {i}"
            assert torch.equal(buf[HEAD + n:], tail), f"{what}: store past the end of allocation {i}"
        del allocs[n0:]

    def _record(self, eng, op, role, x_shape, Co, kind, **kw):
        net = self.net[id(eng)]
        key = (net, role, tuple(x_shape), Co)
        want, block = self.table.get(key, (None, None))
        rec = dict(op=op, net=net, role=role, block=block, key=key, kind=kind, x_shape=tuple(x_shape), **kw)
        assert want is not None, f"call {len(self.calls)}: {key} is not in the table of tests/test_train_calls_cpu.py"
        assert kind == want, f"call {len(self.calls)}: {key} ran {kind}, the table says {want}"
        if kind == "simt":
            assert (net, role, block) in SIMT_BY_DESIGN, f"{key}: a bf16 call fell back to the CUDA-core conv"
        return rec

    def _control(self, family, out, wrong, dtype, acc, what):
        """A negative control: the bound rejects the perturbed reference (once per family)."""
        if family not in self.controls:
            _rejects(out, wrong, dtype, acc, f"{what}: {family}")
            self.controls[family] = what

    # ---------------------------------------------------------------- Engine.conv
    def _ta(self, eng, x, pk, kw, y):
        return eng._tc_args(x, pk, tuple(kw.get("stride", (1, 1, 1))), kw.get("pad"), kw.get("out_spatial"),
                            kw.get("act", ACT_NONE), kw.get("shuffle", SHUFFLE_NONE), False, res=kw.get("res"), y=y)

    def conv(self, eng, x, pk, **kw):
        orig = self.orig[(id(eng), "conv")]
        if self.nested is not None:         # the conv of a data gradient: the dgrad wrapper checks it
            kind, y = _ran(eng, lambda: orig(x, pk, **kw))
            self.nested.update(kind=kind, pk=pk, ta=self._ta(eng, x, pk, kw, y))
            return y
        n0 = len(self.guard[id(eng)].allocs)
        kind, y = _ran(eng, lambda: orig(x, pk, **kw))
        role = self.roles.get(id(pk))
        what = f"call {len(self.calls)}: {self.net[id(eng)]} {role} x {tuple(x.shape)} -> {tuple(y.shape)} on {kind}"
        self._done(eng, n0, what)
        assert role is not None, f"{what}: a conv with a pack the discriminator / VGG do not own"
        kt, kh, kw_ = pk.k_tc or pk.k
        rec = self._record(eng, "conv", role, x.shape, pk.Co, kind, pk=pk, y_shape=tuple(y.shape),
                           stride=tuple(kw.get("stride", (1, 1, 1))), pad=tuple(kw.get("pad") or (kt - 1, kh // 2, kw_ // 2)),
                           out_sp=tuple(kw.get("out_spatial") or x.shape[1:4]), act=kw.get("act", ACT_NONE),
                           res=kw.get("res") is not None)
        if kind == "slab":
            rec["plan"] = _lib_plan(self.lib, self._ta(eng, x, pk, kw, y), self.n_sm)
        if role.endswith("_kw"):
            rec["video"] = self.ingest.pop(id(eng))
        self._check_conv(rec, x, y, kw.get("res"), video=rec.get("video"), controls=True)
        rec.pop("video", None)
        self.calls.append(rec)
        return y

    def _module(self, rec):
        """The module a forward conv's reference is built from."""
        blocks = self.d.blocks
        if rec["role"] == "net0_kw":
            return blocks[0][0].net[0]
        if rec["role"] == "down":
            return blocks[rec["block"]][0].downsample[1]
        if rec["role"] == "logits_lin":
            return self.d.to_logits[3]
        if rec["role"] == "conv_kw":
            return self.vgg.features[0]
        return [m for m in self.vgg.classifier if isinstance(m, torch.nn.Linear)][int(rec["role"][6]) - 1]

    def _check_conv(self, rec, x, y, res, exact=False, w=None, b=None, video=None, controls=False, defects=False):
        """One conv against its float64 reference; w / b: the (grid) weights of a replay, else the pack's / module's."""
        pk, role, kind, B = rec["pk"], rec["role"], rec["kind"], rec["x_shape"][0]
        what = f"{rec['net']} {role} x {rec['x_shape']} on {kind}" + (" (replay)" if exact else "")
        if role == "fc1":                 # fc1 + GEGLU; the hidden channels pack_ff pads in are exactly zero
            w1 = pk.w.double()[0].T if w is None else w
            b1 = pk.bias.double() if b is None else b
            I = w1.shape[0] // 2
            assert torch.equal(y[..., I:].float(), torch.zeros_like(y[..., I:].float())), f"{what}: padded channels"
            for i in range(B):
                ref, acc, _ = geglu64(x[i:i + 1].double(), w1, b1, kind, exact=exact)
                _check(y[i:i + 1, ..., :I], ref, BF, acc, f"{what}, image {i}")
            return
        if role in ("logits_lin", "linear1") and w is None:
            return self._check_map_linear(rec, x, y)
        if role in ("linear1_t", "linear2_t") and w is None:
            return self._check_linear_t(rec, x, y)
        stride, pad, out_sp, act, mode = rec["stride"], rec["pad"], rec["out_sp"], rec["act"], pk.epi_mode
        if role.endswith("_kw"):          # the images (rounded to bf16 as mv2_ingest_kwpack reads them), the module's 3x3
            if w is None:
                mod = self._module(rec)
                w, b = mod.weight.double()[:, :, None], mod.bias.double()
            xs = lambda i: video[i:i + 1].to(BF).double().permute(0, 2, 3, 4, 1)
            pad, K = (0, 1, 1), KW_K
        elif role == "down":              # the module's 1x1 conv on F.pixel_unshuffle of the input
            if w is None:
                mod = self._module(rec)
                w, b = mod.weight.double(), mod.bias.double()
            w = w.reshape(*w.shape, 1) if w.dim() == 4 else w
            xs = lambda i: F.pixel_unshuffle(_cf(x[i:i + 1]), 2).permute(0, 2, 3, 1)[:, None]
            stride, pad, K = (1, 1, 1), (0, 0, 0), w.shape[1]
        else:
            if w is None:
                w = pk.w.double().permute(2, 1, 0).reshape(pk.Co, pk.Ci, *pk.k)
                b = pk.bias.double() if pk.bias is not None else torch.zeros(pk.Co, device="cuda", dtype=torch.float64)
            xs = lambda i: x[i:i + 1, ..., :pk.Ci].double()
            K = math.prod(pk.k) * pk.Ci
        kw = dict(kern=kind, stride=stride, pad=pad, out_sp=out_sp, K=K, act=act, mode=mode)
        for i in range(B):
            r = None if res is None else res[i:i + 1].double()
            ref, acc = forward64(xs(i), w, b, None, r, dtype=BF, exact=exact, **kw)
            _check(y[i:i + 1], ref, BF, acc, f"{what}, image {i}")
            if controls and i == 0 and act == ACT_LEAKY_RELU:
                z, _ = forward64(xs(i), w, b, None, None, dtype=BF, exact=exact, **dict(kw, act=ACT_NONE))
                self._control("LeakyReLU slope 0.2", y[:1], F.leaky_relu(z, 0.2), BF, acc, what)
            if controls and i == 0 and mode == 2:
                wrong, _ = forward64(xs(i), w, b, None, r, dtype=BF, exact=exact,
                                     wrong="scaled-residual factor applied before the residual add", **kw)
                self._control("the 2^-0.5 scale on one branch only", y[:1], wrong, BF, acc, what)
            del ref, acc
        if defects and kind == "slab":
            rec["rejected"] = self._slab_defects(rec, xs, w, b, y, kw, res)
        elif defects and kind == "tap":
            if role == "down":            # the kernel's GEMM is the 2x2 stride-2 conv: its K chunk is 64 channels of one tap
                conv_form = (unshuffle_conv_weight(w[:, :, 0]).unsqueeze(2), (1, 2, 2), (0, 0, 0))
            else:
                conv_form = (w, stride, pad)
            rec["rejected"] = self._tap_defect(rec, xs, w, b, y, kw, res, x[..., :pk.Ci_tc].double(), *conv_form)

    def _check_map_linear(self, rec, x, y):
        """to_logits' Linear / the VGG's first Linear (the average pool folded in) against the module (docstring)."""
        lin = self._module(rec)
        W, b = lin.weight.double(), lin.bias.double()
        h, ha = _cf(x), _cf(x).abs()
        what = f"{rec['net']} {rec['role']} x {rec['x_shape']} on {rec['kind']}"
        K = math.prod(rec["pk"].k) * rec["pk"].Ci
        B = x.shape[0]
        if rec["role"] == "logits_lin":
            z, S = F.linear(h.flatten(1), W, b), F.linear(ha.flatten(1), W.abs())
            acc = _gamma(K, C_OF[rec["kind"]]) * S + 3 * U * (S + b.abs())
            _check(y.reshape(B, -1), z, BF, acc, what)
            wrong = F.linear(h.permute(0, 2, 3, 1).flatten(1), W, b)           # the weight read in (h w c) order
            self._control("the logits weight read in (h w c) order", y.reshape(B, -1), wrong, BF, acc, what)
            return
        oh, ow = self.vgg.avgpool.output_size

        def lin64(pool_of):
            return F.linear(pool_of(h).flatten(1), W, b), F.linear(pool_of(ha).flatten(1), W.abs())
        z, S = lin64(lambda t: F.adaptive_avg_pool2d(t, (oh, ow)))
        acc = _gamma(K, C_OF[rec["kind"]]) * (1 + 2.0 ** -7) * S + 3 * U * (S + b.abs()) + FOLD * S
        _check(y.reshape(B, -1), F.relu(z), BF, acc, what)
        fmap = tuple(x.shape[2:4])

        def shifted(t):                   # every averaging window one input position later (wrapping around)
            ah, aw = (adaptive_pool_matrix(n, o).to(t.device).roll(1, dims=1) for n, o in zip(fmap, (oh, ow)))
            return torch.einsum("bchw,yh,xw->bcyx", t, ah, aw)
        zw, _ = lin64(shifted)
        self._control("the average-pool windows shifted by one", y.reshape(B, -1), F.relu(zw), BF, acc, what)

    def _check_linear_t(self, rec, x, y):
        """The VGG's transposed Linears (data gradients) against the float64 product with the Linear's weight."""
        lin = self._module(rec)
        W = lin.weight.double()
        B = x.shape[0]
        g = x.reshape(B, -1).double()
        gx, S = g @ W, g.abs() @ W.abs()
        K = rec["pk"].Ci
        what = f"vgg {rec['role']} x {rec['x_shape']} on {rec['kind']}"
        if rec["role"] == "linear2_t":
            _check(y.reshape(B, -1), gx, BF, _gamma(K, C_OF[rec["kind"]]) * S, what)
            return
        fmap, c_last = self.m._vgg_cache.packs["fmap"], self.m._vgg_cache.packs["c_last"]
        out_size = self.vgg.avgpool.output_size
        gm = _pool_adjoint(gx.reshape(B, c_last, *out_size), fmap, out_size).permute(0, 2, 3, 1)
        Sm = _pool_adjoint(S.reshape(B, c_last, *out_size), fmap, out_size).permute(0, 2, 3, 1)
        acc = (_gamma(K, C_OF[rec["kind"]]) * (1 + 2.0 ** -7) + FOLD) * Sm
        _check(y.reshape(B, *fmap, c_last), gm, BF, acc, what)

    # ---------------------------------------------------------------- pipeline defects of the replays
    def _slab_defects(self, rec, xs, w, b, y, kw, res=None):
        """_defect_deltas at the schedule's last tile; where every CTA runs one tile only the ring-stage defect exists."""
        plan = rec["plan"]
        if plan["total"] > plan["grid"]:
            deltas = _defect_deltas(self.lib, rec["ta"], self.n_sm, xs, w, kw["pad"], kw["out_sp"], None, plan)
        else:
            out = (C.c_int32 * 6)()
            assert self.lib.mv2_tc_slab_tile(C.byref(rec["ta"]), self.n_sm, last_cta(plan["total"], plan["grid"]), 0, out) == 0
            last = tuple(out)
            assert last[0] == plan["total"] - 1
            kt, kh, kw_ = w.shape[2:]
            ws = torch.zeros_like(w)
            ws[:, :64, kt - 1, kh // 2, kw_ // 2] = w[:, :64, kt - 1, kh // 2, kw_ // 2]
            stage = _acc64(xs(last[1]), ws, kw["pad"], kw["out_sp"], None)
            d = torch.zeros_like(stage)
            r = _region(last, plan, stage.shape)
            d[r] = -stage[r]
            deltas = {"one ring stage missing": (last[1], d)}
        for defect, (i, delta) in deltas.items():
            r = None if res is None else res[i:i + 1].double()
            ref, acc = forward64(xs(i), w, b, None, r, dtype=BF, exact=True, **kw)
            wrong, _ = forward64(xs(i), w, b, None, r, dtype=BF, exact=True, delta=delta, **kw)
            _rejects(y[i:i + 1], wrong, BF, acc, f"{rec['key']}: {defect}")
        return sorted(deltas)

    def _tap_defect(self, rec, xs, w, b, y, kw, res, x, wc, stride, pad):
        """Input channels 0..63 of the last tap of the kernel's conv (x, wc, stride, pad) missing from every accumulator:
        one K chunk of the tap-wise kernel."""
        kt, kh, kw_ = wc.shape[2:]
        ws = torch.zeros_like(wc)
        ws[:, :64, kt - 1, kh - 1, kw_ - 1] = wc[:, :64, kt - 1, kh - 1, kw_ - 1]
        x_all = torch.cat([xs(i) for i in range(rec["x_shape"][0])])
        r = None if res is None else res.double()
        ref, acc = forward64(x_all, w, b, None, r, dtype=BF, exact=True, **kw)
        delta = -_conv64(x, ws, stride, pad, kw["out_sp"])
        assert delta.abs().max() > 0
        wrong, _ = forward64(x_all, w, b, None, r, dtype=BF, exact=True, delta=delta, **kw)
        _rejects(y, wrong, BF, acc, f"{rec['key']}: one 64-channel K chunk missing")
        return ["one K chunk missing"]

    # ---------------------------------------------------------------- data gradients
    def _dgrad_wrapper(self, fn, op):
        rec_ = self

        def wrapped(runner, g, w, *args):
            eng = runner.eng
            if id(eng) not in rec_.net:       # the tokenizer's runner: tests/test_train_tokenizer_calls_gpu.py
                return fn(runner, g, w, *args)
            n0 = len(rec_.guard[id(eng)].allocs)
            rec_.nested = inner = {}
            try:
                out = fn(runner, g, w, *args)
            finally:
                rec_.nested = None
            what = f"call {len(rec_.calls)}: {rec_.net[id(eng)]} {op} g {tuple(g.shape)} on {inner.get('kind')}"
            rec_._done(eng, n0, what)
            rec_.check_dgrad(eng, runner, op, g, w, args, out, inner)
            return out
        return wrapped

    def _s2_weight(self, wd):
        """(module weight, stride2_1x1) whose builder made the stride-2 dgrad weights wd."""
        for block, _ in self.d.blocks:
            cr, ds = block.conv_res, block.downsample
            if ds is not None and wd.shape == unshuffle_dgrad_weight(ds[1].weight).shape and torch.equal(
                    wd, unshuffle_dgrad_weight(ds[1].weight.detach())):
                return ds[1].weight, False
            if cr.stride == (2, 2) and wd.shape[0] == 4 * cr.weight.shape[1] and torch.equal(
                    wd, stride2_1x1_dgrad_weight(cr.weight.detach())):
                return cr.weight, True
        raise AssertionError("stride-2 dgrad weights no discriminator module builds")

    def check_dgrad(self, eng, runner, op, g, w, args, out, inner, exact=False, w_mod=None):
        pk, kind = inner["pk"], inner["kind"]
        if op == "dgrad":
            k, out_spatial = args[0], tuple(args[1])
            role, Co = f"dgrad k{k[1]}{k[2]}", w.shape[1]
        else:
            role, Co = "dgrad_s2", w.shape[0]
        rec = self._record(eng, op, role, g.shape, Co, kind, pk=pk, ta=inner["ta"], runner=runner, w_shape=tuple(w.shape),
                           args=args)
        if kind == "slab":
            rec["plan"] = _lib_plan(self.lib, inner["ta"], self.n_sm)
        what = f"{rec['key']} on {kind}" + (" (replay)" if exact else "")
        B = g.shape[0]
        for i in range(B):
            gi = g[i:i + 1]
            if op == "dgrad":
                ref = _dgrad64(gi, w, k, out_spatial)
                acc = 0 if exact else _gamma(w.shape[0] * math.prod(k), C_OF[kind]) * _dgrad64(gi.abs(), w.abs(), k, out_spatial)
            else:
                wm, one = (self._s2_weight(w) if w_mod is None else w_mod)
                rec["s2"] = (tuple(wm.shape), one)
                hw = tuple(args[0][2:4])
                ref = _s2_grad64(gi, wm, one, hw)
                acc = 0 if exact else _gamma(g.shape[-1], C_OF[kind]) * _s2_grad64(gi.abs(), wm.abs(), one, hw)
                if not one and i == 0:
                    wrong = ref.reshape(1, 1, hw[0] // 2, 2, hw[1] // 2, 2, -1).transpose(3, 5).reshape(ref.shape)
                    self._control("the depth-to-space phases swapped", out[:1], wrong, BF, acc, what)
            _check(out[i:i + 1], ref, out.dtype, acc, f"{what}, image {i}")
            del ref, acc
        if not exact:
            self.calls.append(rec)
        return rec

    # ---------------------------------------------------------------- the CUDA-core ops
    def ingest_kwpack(self, eng, v, t_pad, pin):
        n0 = len(self.guard[id(eng)].allocs)
        out = self.orig[(id(eng), "ingest_kwpack")](v, t_pad, pin)
        what = f"call {len(self.calls)}: {self.net[id(eng)]} ingest_kwpack {tuple(v.shape)}"
        self._done(eng, n0, what)
        B, C_, T, H, W = v.shape
        kw, pw = pin.kw_orig, pin.kw_orig // 2
        xp = F.pad(v.double().permute(0, 2, 3, 4, 1), (0, 0, pw, kw - 1 - pw, 0, 0, t_pad, 0))
        want = torch.zeros(out.shape, device="cuda", dtype=torch.float64)
        for dw in range(kw):
            want[..., dw * C_:(dw + 1) * C_] = xp[:, :, :, dw:dw + W]
        assert torch.equal(out.double(), want.to(BF).double()), what
        self.ingest[id(eng)] = v
        self.calls.append(dict(op="ingest", net=self.net[id(eng)], kind="simt"))
        return out

    def rmsnorm(self, eng, x, gamma, token_shift=False, ss=None):
        assert ss is None and not token_shift
        n0 = len(self.guard[id(eng)].allocs)
        out = self.orig[(id(eng), "rmsnorm")](x, gamma)
        what = f"call {len(self.calls)}: {self.net[id(eng)]} rmsnorm {tuple(x.shape)}"
        self._done(eng, n0, what)
        B, T, H, W, C_ = x.shape
        ref = _rms_ref(x.double().reshape(B, T, H * W, C_), gamma.double(), False)
        depth = -(-C_ // 32) + 5
        _check(out.reshape(B, T, H * W, C_), ref, BF, (depth + 6) * U * ref.abs(), what)
        self.calls.append(dict(op="rmsnorm", net=self.net[id(eng)], kind="simt"))
        return out

    def maxpool2x2(self, eng, x):
        n0 = len(self.guard[id(eng)].allocs)
        y = self.orig[(id(eng), "maxpool2x2")](x)
        what = f"call {len(self.calls)}: maxpool2x2 {tuple(x.shape)}"
        self._done(eng, n0, what)
        assert torch.equal(_cf(y), F.max_pool2d(_cf(x), 2, 2)), what
        self.calls.append(dict(op="maxpool", net=self.net[id(eng)], kind="simt"))
        return y

    def maxpool2x2_backward(self, eng, g, x):
        n0 = len(self.guard[id(eng)].allocs)
        gx = self.orig[(id(eng), "maxpool2x2_backward")](g, x)
        what = f"call {len(self.calls)}: maxpool2x2_backward {tuple(x.shape)}"
        self._done(eng, n0, what)
        gb = g.to(x.dtype)
        assert torch.equal(gx.double(), _pool_grad64(gb, x)), what
        # a tie between positive maxima sending its gradient to the last maximum differs (counted over the step's pools)
        self.calls.append(dict(op="maxpool_bwd", net=self.net[id(eng)], kind="simt",
                               tie_rejected=not torch.equal(gx.double(), _pool_grad64(gb, x, last=True))))
        return gx

    def mse(self, eng, a, b):
        n0 = len(self.guard[id(eng)].allocs)
        out = self.orig[(id(eng), "mse")](a, b)
        what = f"call {len(self.calls)}: mse {tuple(a.shape)}"
        self._done(eng, n0, what)
        a64, b64 = a.double().flatten(), b.double().flatten()
        n = a64.numel()
        dl = a64 - b64
        ref = (dl * dl).mean()
        steps = -(-n // (min(592, -(-n // 256)) * 256))
        tol = (steps + 6) * U * ref + 3 * U * (a64.abs() * dl.abs()).mean()
        assert abs(out.double().item() - ref.item()) <= tol.item(), (what, out.item(), ref.item())
        self.calls.append(dict(op="mse", net=self.net[id(eng)], kind="simt"))
        return out

    # ---------------------------------------------------------------- exact replay
    def replay(self, rec, gen, defects):
        """The call again on REPLAY_GRID operands with the same packer, entry point and arguments (module docstring)."""
        if rec["op"] != "conv":
            return self._replay_dgrad(rec, gen, defects)
        pk, role = rec["pk"], rec["role"]
        eng = self.d._pack_cache.engine if rec["net"] == "discr" else self.m._vgg_cache.engine
        conv = self.orig[(id(eng), "conv")]
        kw = dict(stride=rec["stride"], pad=rec["pad"], out_spatial=rec["out_sp"], act=rec["act"])
        video = res = None
        if role.endswith("_kw"):
            w, b = _grid((pk.Co, 3, 3, 3), "w", gen), _grid(pk.Co, "b", gen)
            pk2 = pack_conv_in_kwpack(w[:, :, None].float(), b.float())
            B, _, H, W, _ = rec["x_shape"]
            video = _grid((B, 3, 1, H, W), "x", gen)
            x = self.orig[(id(eng), "ingest_kwpack")](video.to(BF), 0, pk2)
            w = w[:, :, None]
        elif role in ("fc1", "fc2"):      # pack_ff
            C_, I = (pk.Ci, pk.Co // 2) if role == "fc1" else (pk.Co, pk.Ci)
            w1, b1 = _grid((2 * I, C_), "w", gen), _grid(2 * I, "b", gen)
            w2, b2 = _grid((C_, I), "w", gen), _grid(C_, "b", gen)
            fc1, fc2 = pack_ff(w1.float()[..., None, None, None], b1.float(), w2.float()[..., None, None, None], b2.float(), BF)
            pk2 = fc1 if role == "fc1" else fc2
            w, b = (w1, b1) if role == "fc1" else (w2[..., None, None, None], b2)
            x = _grid(rec["x_shape"][:-1] + (pk2.Ci_tc,), "x", gen)
        elif role == "down":              # the module's 1x1 weight through unshuffle_conv_weight
            Co = pk.Co
            w, b = _grid((Co, 4 * pk.Ci, 1, 1), "w", gen), _grid(Co, "b", gen)
            pk2 = pack_conv(unshuffle_conv_weight(w).float(), b.float(), BF)
            x = _grid(rec["x_shape"], "x", gen)
        else:
            w, b = _grid((pk.Co, pk.Ci, *pk.k), "w", gen), _grid(pk.Co, "b", gen)
            if pk.bias is None:
                b = torch.zeros_like(b)
            pk2 = pack_conv(w.float(), None if pk.bias is None else b.float(), BF, k=pk.k)
            x = _grid(rec["x_shape"], "x", gen)
        pk2.epi_mode = pk.epi_mode
        if rec["res"]:
            res = _grid(rec["y_shape"], "x", gen)
            kw["res"] = res.to(BF).contiguous()
        n0 = len(self.guard[id(eng)].allocs)
        xb = x.to(BF).contiguous()
        kind, y = _ran(eng, lambda: conv(xb, pk2, **kw))
        self._done(eng, n0, f"replay of {rec['key']}")
        assert kind == rec["kind"], f"replay of {rec['key']}: ran {kind}"
        rec2 = dict(rec, pk=pk2)
        if kind == "slab":
            rec2["ta"] = self._ta(eng, xb, pk2, kw, y)
        self._check_conv(rec2, x, y, res, exact=True, w=w, b=b, video=video,
                         defects=defects and role != "fc1" and not role.endswith("_kw"))
        return rec2.get("rejected", [])

    def _replay_dgrad(self, rec, gen, defects):
        runner, eng = rec["runner"], rec["runner"].eng
        g = _grid(rec["x_shape"], "x", gen)
        n0 = len(self.guard[id(eng)].allocs)
        self.nested = inner = {}
        try:
            if rec["op"] == "dgrad":
                w = _grid(rec["w_shape"], "w", gen)
                out = self.orig_dgrad(runner, g.to(BF).contiguous(), w.to(BF), *rec["args"])
                w_mod = None
            else:
                shape, one = rec["s2"]
                w = _grid(shape, "w", gen)
                wd = (stride2_1x1_dgrad_weight if one else unshuffle_dgrad_weight)(w.to(BF))
                out = self.orig_s2(runner, g.to(BF).contiguous(), wd, *rec["args"])
                w_mod = (w, one)
        finally:
            self.nested = None
        self._done(eng, n0, f"replay of {rec['key']}")
        assert inner["kind"] == rec["kind"], f"replay of {rec['key']}: ran {inner['kind']}"
        rec2 = self.check_dgrad(eng, runner, rec["op"], g, w if rec["op"] == "dgrad" else wd, rec["args"], out, inner,
                                exact=True, w_mod=w_mod)
        if not (defects and rec["op"] == "dgrad" and inner["kind"] == "slab"):
            return []
        pk = inner["pk"]                  # the transposed conv the kernel ran, for the defect's accumulators
        wt = pk.w.double().permute(2, 1, 0).reshape(pk.Co, pk.Ci, *pk.k)
        k = rec["args"][0]
        kw = dict(kern="slab", stride=(1, 1, 1), pad=(0, k[1] // 2, k[2] // 2), out_sp=tuple(rec["args"][1]),
                  K=math.prod(pk.k) * pk.Ci, act=ACT_NONE, mode=0)
        rec2["ta"] = inner["ta"]
        return self._slab_defects(rec2, lambda i: g[i:i + 1], wt, torch.zeros(pk.Co, device="cuda", dtype=torch.float64),
                                  out, kw)


def _counts(calls):
    """Calls per (network, kind), in the kinds of tests/test_train_calls_cpu.step_counts."""
    out = {}
    for c in calls:
        k = "linear_t" if c.get("role", "").endswith("_t") else c["op"]
        out[(c["net"], k)] = out.get((c["net"], k), 0) + 1
    return out


CONTROLS = {"LeakyReLU slope 0.2", "the 2^-0.5 scale on one branch only", "the logits weight read in (h w c) order",
            "the average-pool windows shifted by one", "the depth-to-space phases swapped"}
STAGE, RESET, CHUNK = "one ring stage missing", "previous tile's accumulators not reset", "one K chunk missing"


def test_readme_train_step_calls_vs_float64(monkeypatch):
    t0 = time.time()
    m = _model()
    video = synth_data.synth_video(CLIPS, 3, 17, 128).cuda().bfloat16()
    torch.manual_seed(1)                  # the frame picks draw from torch's CPU generator
    loss, _ = m(video, return_loss=True)  # warm-up: the discriminator's and the VGG's packs and engines
    loss.backward()
    del loss
    rec = _Recorder(monkeypatch, m)
    # ---- the generator step ----
    torch.manual_seed(2)
    loss, _ = m(video, return_loss=True)
    loss.backward()
    del loss
    gen_calls, rec.calls = rec.calls, []
    # ---- the discriminator step ----
    torch.manual_seed(3)
    loss, _ = m(video, return_discr_loss=True, apply_gradient_penalty=False)
    loss.backward()
    del loss
    torch.cuda.synchronize()
    dis_calls = rec.calls
    # ---- structure: calls per kind, kernels, tiles per CTA, negative controls ----
    want_gen, want_dis = step_counts(m)
    assert _counts(gen_calls) == want_gen, (_counts(gen_calls), want_gen)
    assert _counts(dis_calls) == want_dis, (_counts(dis_calls), want_dis)
    calls = gen_calls + dis_calls
    seen = {c["key"] for c in calls if "key" in c}
    assert seen == set(rec.table), (set(rec.table) - seen, seen - set(rec.table))
    for eng_id in rec.net:
        eng = rec.d._pack_cache.engine if rec.net[eng_id] == "discr" else m._vgg_cache.engine
        assert eng.simt_conv_calls - rec.simt0[eng_id] == sum(c["kind"] == "simt" and c["op"] in ("conv", "dgrad", "dgrad_s2") and
                                          c["net"] == rec.net[eng_id] for c in calls)
    big = [c for c in calls if c["kind"] == "slab" and c["x_shape"][2] == 128]
    assert big and all(c["plan"]["total"] > c["plan"]["grid"] for c in big), [(c["key"], c["plan"]) for c in big]
    wide = [c for c in big if c["net"] == "discr" and c["key"][3] == 512]
    assert wide and all(c["plan"]["total"] > 2 * c["plan"]["grid"] for c in wide)
    assert set(rec.controls) == CONTROLS, set(rec.controls)
    assert any(c.get("tie_rejected") for c in calls), "no pool backward had a tie between positive maxima"
    # ---- exact replay of every distinct wgmma call; the pipeline defects on each ----
    gen = torch.Generator(device="cuda").manual_seed(7)
    rejected = {}
    for c in calls:
        if c["op"] not in ("conv", "dgrad", "dgrad_s2") or c["kind"] == "simt" or c["key"] in rejected:
            continue
        rejected[c["key"]] = (c["kind"], c.get("plan"), rec.replay(c, gen, defects=True))
    for eng_id, guard in rec.guard.items():
        eng = rec.d._pack_cache.engine if rec.net[eng_id] == "discr" else m._vgg_cache.engine
        rec._done(eng, 0, "allocations outside the checked calls")
    n_tap = n_slab = 0
    for key, (kind, plan, got) in rejected.items():
        if kind == "tap":
            assert got == [CHUNK], (key, got)
            n_tap += 1
        elif key[1] in ("fc1", "dgrad_s2", "net0_kw", "conv_kw"):
            assert got == [], (key, got)
        else:
            assert got == sorted([STAGE, RESET] if plan["total"] > plan["grid"] else [STAGE]), (key, plan, got)
            n_slab += 1
    # the calls the replay must reach: both depth-8192 tap calls, the 4096-deep 1x1 calls, the 3x3 slab calls on the
    # 4 x 4 map, the 3-channel image data gradients
    must = {("discr", "logits_lin"): CHUNK, ("vgg", "linear1"): CHUNK, ("vgg", "linear1_t"): CHUNK,
            ("vgg", "linear2"): STAGE, ("vgg", "linear2_t"): STAGE}
    for (net, role), defect in must.items():
        assert any(k[:2] == (net, role) and defect in v[2] for k, v in rejected.items()), (net, role)
    for role in ("net0", "net2", "logits_conv", "dgrad k33"):
        assert any(k[:2] == ("discr", role) and k[2][2] == 4 and STAGE in v[2] for k, v in rejected.items()), role
    for net, Ci in (("discr", 512), ("vgg", 64)):
        k = (net, "dgrad k33", (CLIPS, 1, 128, 128, Ci), 3)
        assert set(rejected[k][2]) == {STAGE, RESET}, (k, rejected[k])
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"\n{len(gen_calls)} generator-step and {len(dis_calls)} discriminator-step calls checked; {len(rejected)} "
          f"distinct wgmma calls replayed ({n_tap} tap, {n_slab} slab with defects); controls rejected: "
          f"{sorted(rec.controls.items())}; wall {time.time() - t0:.0f} s, peak device memory "
          f"{peak:.1f} GiB")
