"""The forward conv kernels' epilogues, strided and fused variants against plain float64 torch references: the slab kernel
(tc_slab.cu) and its down-space variant, the tap-wise wgmma kernel (tc_conv.cu), the CUDA-core conv (conv_simt_kernel,
simt_ops.cu) and the fused ResidualUnit (mv2_tc_ru_forward + mv2_se_gate_records), at the tile, stride, shuffle and
frame edges where an epilogue goes wrong.

  1. slab epilogues: EPI_PLAIN (every activation, bn = 32 / 64 / 128 and the ragged 128-column last tile of a wide
     output, mw = 1 / 2 / 4 with W not a multiple of 8 mw, H not a multiple of 16, T = 1, 64-byte rows, per-clip oscale),
     EPI_PLAIN_RES (epi_mode 0 / 2, oscale), EPI_RAGGED (Co = 3 / 13, oscale, the channels-first conv_out store with a
     leading-frame crop of 0 / 1 / 3 frames), EPI_SHUFFLE_ST, EPI_SHUFFLE, EPI_GEGLU (pack_ff and hand-packed widths) and
     the time-strided slab;
  2. the down-space slab (and an odd plane falling back to the tap-wise kernel);
  3. the tap-wise kernel: bk = 16 / 32 / 64, bn = 32 / 64 / 128 with ragged last N tiles, its three output-box regimes,
     a K loop shorter than the ring, strides (1,2,2) and (2,1,1) with odd extents, every epilogue flavour;
  4. the kw-packed conv_in (Engine.ingest_kwpack + the 7x7x7 conv) on the slab and the tap-wise kernel;
  5. the CUDA-core conv in bf16 and fp32: ragged M / Co, Ci = 3 / 5 / 48, token shift with odd Ci, shuffles, strides,
     oscale, residual, every activation and the two-rounding epi_mode 2 path;
  6. the fused ResidualUnit's y and its SqueezeExcite gates.

Every call goes through Engine.conv / Engine.residual_unit with the engine's allocator wrapped (fixture `guarded`): each
output is NaN-filled before the call, so an element the kernel never writes fails, and sits between a head and a tail
sentinel that must come back unchanged, so a stray store outside the tensor fails as silent corruption would.  Each case
asserts from the engine's counters (and conv_log) which kernel ran, and a slab case the plan (mw, bn, n_tiles_n,
slab_stages) of mv2_tc_slab_plan it claims to exercise.

References.  Inputs, weights, residuals are bf16-representable; bias and oscale are fp32 values.  The reference runs in
float64 on the device: F.conv3d with the kernels' zero padding (frame / row / column o*s - p + d, zero outside), the exact
activation (ELU, SiLU, leaky_relu(0.1), ReLU, erf-GELU), the reference modules' (c p1 p2) / (c p) shuffles.

Per-element bound: half an ulp of the output dtype at the reference value (_check) plus an allowance `acc`:
  * accumulation: gamma_c(K) * S with S = (|W| (*) |x|) (the same conv of absolute values), K the GEMM depth (taps x Ci of
    the packed GEMM), gamma_c(K) = c K u / (1 - c K u), u = 2^-24; c = 1 for the CUDA-core conv's round-to-nearest fma
    chains, c = 2 for wgmma, whose fp32 additions may truncate (see tests/test_conv_grad_gpu.py);
  * oscale: S scaled by |oscale|, plus one fp32 rounding for the oscale product and one for the bias add:
    e_pre = gamma S |os| + 3 u (S |os| + |b|);
  * activation: e_pre times the activation's largest slope (1; SiLU 1.0998 -> 1.1; GELU 1.129 -> 1.13), plus the error
    of its evaluation.  wgmma epilogues use the MUFU forms of tc_common.cuh: ex2.approx.ftz.f32 has a maximum error of
    2 ulp over its full range and rcp.approx.ftz.f32 1 ulp (PTX ISA, "Floating-point instructions: ex2 / rcp"), i.e.
    relative 2^-22 and 2^-23; flush-to-zero adds at most 2^-126 absolute.  ELU(z < 0) = ex2(z log2 e) - 1 is then within
    2^-22 + 3u absolute (e^z <= 1, |z| e^z <= 1/e bounds the argument's rounding); SiLU = z rcp(1 + ex2(-z log2 e)) within
    |v| (2^-22 + 2^-23 + 4u) + u v^2; gelu_fast (Abramowitz & Stegun 7.1.26, |erf error| <= 1.5e-7, so
    |Phi error| <= 0.75e-7) within |g| (0.75e-7 + 0.5 (2^-22 + 2 2^-23 + 8u + u g^2)) + u |gelu|.  The CUDA-core conv uses
    expm1f / expf and IEEE division: within 8u |v|;
  * residual: one fp32 rounding of act + res (u |act + res|); epi_mode 2 multiplies by fp32(2^-0.5) (relative error
    < u) and rounds: (e + u |t|) s + 2u |ref|;
  * GEGLU: |x| (e_gelu + 1.13 e_gate) + |gelu(gate)| e_x + u |out|.
The wgmma epilogues round once (tc_common.cuh epi_chunk32_t, tc_slab.cu EPI_PLAIN_RES).  The CUDA-core epi_mode 2 path
rounds twice (conv + residual rounded to the output dtype, then mv2_scale_channels): its reference is the float64
(act + res) 2^-0.5 and its bound covers the first rounding, s (half an ulp at |t| + e) added to e.

Fused ResidualUnit: y = ELU(conv1(round_bf16(ELU(conv3 x + b3))) + b1).  The kernel rounds h to bf16 in shared memory; an
h element whose float64 value lies within its own allowance of a bf16 rounding boundary may round either way, so for
exactly those elements |W1| ulp(h) is added to the bound of y.  The gates' reference is the float64 softmax pool, gate
MLP and sigmoid of the kernel's own bf16 y, within the fp32 gate bound of tests/test_simt_ops_gpu.py (GATE_TOL).

Each family shows that its bound rejects a slightly wrong reference: the bias added after the activation, clip 0's oscale
used for clip 1, oscale applied after the bias, the scaled-residual factor applied before the residual add, shuffle phases
p1 / p2 swapped, the GEGLU halves swapped, the down-space / time-down pad at the back, the token shift split at
floor(Ci / 2), the channels-first output cropped one frame late, and the fused RU gates computed without the frame's last
ragged row or without its last column."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_conv_grad_gpu import C_OF, _bfrand, _engine, _gamma, _gen
from tests.test_simt_ops_gpu import GATE_TOL, U, _check, _rejects, _se_gates64, _ulp

from magvit2_pytorch_b200 import _lib
from magvit2_pytorch_b200._lib import (ACT_ELU, ACT_LEAKY_RELU, ACT_NONE, ACT_RELU, ACT_SILU, SHUFFLE_NONE,
                                       SHUFFLE_SPACE, SHUFFLE_TIME, TcConvArgs)
from magvit2_pytorch_b200.engine import ConvPack, pack_conv, pack_conv_down_space, pack_conv_in_kwpack, pack_ff

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "f32": torch.float32}
NONE, ELU, SILU, LEAKY, RELU = ACT_NONE, ACT_ELU, ACT_SILU, ACT_LEAKY_RELU, ACT_RELU
ACT64 = {NONE: lambda v: v, ELU: F.elu, SILU: F.silu, LEAKY: lambda v: F.leaky_relu(v, 0.1), RELU: F.relu}
SLOPE = {NONE: 1.0, ELU: 1.0, SILU: 1.1, LEAKY: 1.0, RELU: 1.0}
R_EX2, R_RCP = 2.0 ** -22, 2.0 ** -23           # ex2.approx / rcp.approx: 2 ulp / 1 ulp relative (PTX ISA)
FTZ = 2.0 ** -126
GELU_SLOPE = 1.13
RS = 2 ** -0.5                                  # the scaled residual's factor (epi_mode 2)
K333, K111, K133 = (3, 3, 3), (1, 1, 1), (1, 3, 3)
N_SM = 132                                      # the plan's grid does not enter (mw, bn, n_tiles_n, slab_stages)
C_KERN = dict(C_OF, down=2, ru=2)              # c of the accumulation allowance per kernel (test_conv_grad_gpu)
HEAD = 4096                                     # sentinel elements in front of every engine allocation


# ------------------------------------------------------------------------------------------------------------------
# guarded allocations and kernel identification
# ------------------------------------------------------------------------------------------------------------------
class _Guard:
    """Engine._new replacement: NaN-filled tensors in the middle of a sentinel-bordered buffer."""

    def __init__(self, eng):
        self.eng, self.allocs = eng, []

    def new(self, shape, dtype=None):
        dtype = dtype or self.eng.dtype
        n = math.prod(shape)
        tail = HEAD + n // 2
        buf = torch.full((HEAD + n + tail,), float("nan"), device=self.eng.device, dtype=dtype)
        g = torch.Generator(device="cuda").manual_seed(len(self.allocs) + 1)
        buf[:HEAD] = torch.randn(HEAD, generator=g, device="cuda").to(dtype)
        buf[HEAD + n:] = torch.randn(tail, generator=g, device="cuda").to(dtype)
        self.allocs.append((buf, n, buf[:HEAD].clone(), buf[HEAD + n:].clone()))
        return buf[HEAD:HEAD + n].view(shape)

    def check_borders(self, what):
        torch.cuda.synchronize()
        for i, (buf, n, head, tail) in enumerate(self.allocs):
            assert torch.equal(buf[:HEAD], head), f"{what}: store before allocation {i}"
            assert torch.equal(buf[HEAD + n:], tail), f"{what}: store past the end of allocation {i}"


@pytest.fixture
def guarded(monkeypatch):
    """guard(eng) -> _Guard: the engine's allocations NaN-filled and sentinel-bordered; conv_log on.  The borders of
    every allocation are checked when the test ends."""
    guards = []

    def guard(eng):
        g = _Guard(eng)
        monkeypatch.setattr(eng, "_new", g.new)
        monkeypatch.setattr(eng, "conv_log", [])
        guards.append(g)
        return g

    yield guard
    for g in guards:
        g.check_borders("guarded allocations")


def _ran(eng, fn):
    """(kernel that ran, result) of one engine call: slab, down (the down-space slab), tap, simt or ru (fused RU)."""
    keys = ("slab_calls", "tc_calls", "simt_conv_calls", "fused_ru_calls")
    c0 = [getattr(eng, k) for k in keys]
    n_log = len(eng.conv_log)
    out = fn()
    d = tuple(getattr(eng, k) - v for k, v in zip(keys, c0))
    kind = {(1, 1, 0, 0): "slab", (0, 1, 0, 0): "tap", (0, 0, 1, 0): "simt", (1, 1, 0, 1): "ru"}.get(d, f"counters moved by {d}")
    if kind in ("slab", "tap"):
        assert len(eng.conv_log) == n_log + 1 and eng.conv_log[-1]["kind"] == kind
        if eng.conv_log[-1]["down_space"]:
            kind = "down"        # a flavour of the slab kernel: counted and logged as "slab", flagged in its record
    return kind, out


def _slab_plan(x_shape, pk, stride, pad, out_sp, shuffle, res, oscale, out_cf):
    """(mw, bn, n_tiles_n, slab_stages) of mv2_tc_slab_plan for the TcConvArgs Engine.conv builds."""
    B, Ti, Hi, Wi, Ci = x_shape
    kt, kh, kw = pk.k_tc
    a = TcConvArgs(x=1, w=1, bias=None, res=1 if res else None, y=1, B=B, Ti=Ti, Hi=Hi, Wi=Wi, Ci=Ci,
                   To=out_sp[0], Ho=out_sp[1], Wo=out_sp[2], Co=pk.Co_tc, kt=kt, kh=kh, kw=kw,
                   st=stride[0], sh=stride[1], sw=stride[2], pt=pad[0], ph=pad[1], pw=pad[2], act=0, shuffle=shuffle,
                   epi_mode=pk.epi_mode, oscale=1 if oscale else None, out_layout=int(out_cf))
    out = (ctypes.c_int32 * 6)()
    lib = _lib.load()
    assert lib.mv2_tc_slab_plan(ctypes.byref(a), N_SM, out) == 0, lib.mv2_last_error()
    return out[0], out[1], out[2], out[5]


# ------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------
def _conv64(x, w, stride, pad, out_sp):
    """x (B,T,H,W,Ci) channels-last float64, w (Co,Ci,kt,kh,kw): y[o] = sum_d w[d] x[o s - p + d], zero outside x (a
    negative p crops), as (B,To,Ho,Wo,Co)."""
    kt, kh, kw = w.shape[2:]
    ext = []
    for n_in, n_out, k, s, p in zip(x.shape[1:4], out_sp, (kt, kh, kw), stride, pad):
        ext.append((p, max(0, (n_out - 1) * s - p + k - n_in)))
    (ft, bt), (fh, bh), (fw, bw) = ext
    xp = F.pad(x.permute(0, 4, 1, 2, 3), (fw, bw, fh, bh, ft, bt))
    y = F.conv3d(xp, w, stride=stride)[:, :, :out_sp[0], :out_sp[1], :out_sp[2]]
    return y.permute(0, 2, 3, 4, 1)


def _act_err(act, z, v, kern):
    """Evaluation error of the activation v = act(z) (see the module docstring)."""
    if act in (ELU, SILU) and kern == "simt":
        return 8 * U * v.abs()
    if act == ELU:
        return torch.where(z < 0, torch.full_like(z, R_EX2 + 3 * U + FTZ), torch.zeros_like(z))
    if act == SILU:
        return v.abs() * (R_EX2 + R_RCP + 4 * U) + U * v * v + FTZ
    return torch.zeros_like(z)


def _gelu_err(g):
    return g.abs() * (0.75e-7 + 0.5 * (R_EX2 + 2 * R_RCP + 8 * U + U * g * g)) + U * F.gelu(g).abs() + FTZ


def _shuffle(y, shuffle, swap=False):
    """The reference's 'b (c p1 p2) h w -> b c (h p1) (w p2)' / 'b (c p) t -> b c (t p)' on channels-last y; `swap`
    exchanges the phases (p1 <-> p2 / p reversed)."""
    if shuffle == SHUFFLE_NONE:
        return y
    B, T, H, W, C_ = y.shape
    if shuffle == SHUFFLE_SPACE:
        y = y.reshape(B, T, H, W, C_ // 4, 2, 2)
        if swap:
            y = y.transpose(5, 6)
        return y.permute(0, 1, 2, 5, 3, 6, 4).reshape(B, T, 2 * H, 2 * W, C_ // 4)
    y = y.reshape(B, T, H, W, C_ // 2, 2)
    if swap:
        y = y.flip(5)
    return y.permute(0, 1, 5, 2, 3, 4).reshape(B, 2 * T, H, W, C_ // 2)


class Case(dict):
    __getattr__ = dict.get


def case(name, kern, **kw):
    d = dict(name=name, kern=kern, dt="bf16", variant="auto", ci=64, co=64, k=K333, shape=(1, 2, 12, 20),
             stride=(1, 1, 1), pad=None, act=NONE, res=False, mode=0, shuffle=SHUFFLE_NONE, oscale=False,
             tshift=False, tp=None, plan=None, down=False)
    d.update(kw)
    return pytest.param(Case(d), id=name)


def _geometry(c):
    """(pad, output spatial extent before any shuffle) of an Engine.conv call of case c."""
    kt, kh, kw = c.k
    B, T, H, W = c.shape
    if c.tp is not None:          # channels-first conv_out: the first tp frames are never computed
        return (kt - 1 - c.tp, kh // 2, kw // 2), (T - c.tp, H, W)
    pad = c.pad if c.pad is not None else (kt - 1, kh // 2, kw // 2)
    st, sh, sw = c.stride
    return pad, ((T + pad[0] - kt) // st + 1, (H + 2 * pad[1] - kh) // sh + 1, (W + 2 * pad[2] - kw) // sw + 1)


def forward64(x, w, b, os, r, *, kern, stride, pad, out_sp, K, act=NONE, mode=0, shuffle=SHUFFLE_NONE, tp=None,
              tshift=False, dtype=torch.bfloat16, wrong=None, exact=False, delta=None):
    """float64 reference and allowance (module docstring) of one Engine.conv call: x (B,T,H,W,Ci) channels-last, w
    (Co,Ci,kt,kh,kw) in the reference's channel order, b (Co,), per-clip oscale `os` (B,Co) or None, residual r or None;
    `pad` / `out_sp` the call's leading pad and output extent before any shuffle, K the packed GEMM depth, `tp` the
    channels-first conv_out's dropped leading frames.  `wrong` names a defect to build into the reference.  `exact`: the
    accumulation and the bias add are exact (operands on a dyadic grid), so only the epilogue's errors are allowed (with
    oscale, the oscale product and the bias add after it round);
    `delta` (B,To,Ho,Wo,Co) is added to the accumulators before the epilogue."""
    kt = w.shape[2]
    if tshift:                    # TokenShift (M:250-254): channels [ceil(C / 2), C) delayed by one frame
        split = x.shape[-1] // 2 if wrong == "token shift split at floor(Ci / 2)" else (x.shape[-1] + 1) // 2
        x = x.clone()
        x[:, 1:, ..., split:] = x[:, :-1, ..., split:].clone()
        x[:, 0, ..., split:] = 0
    if wrong == "pad at the back":
        pad = tuple(0 if s == 2 else p for s, p in zip(stride, pad))
    if tp is not None:            # the full causal conv, then its first tp (or, wrongly, tp + 1) frames dropped
        T = x.shape[1]
        crop = tp + (wrong == "cropped one frame late")
        full = [_conv64(v, wv, (1, 1, 1), (kt - 1,) + pad[1:], (T,) + out_sp[1:]) for v, wv in ((x, w), (x.abs(), w.abs()))]
        acc, S = (torch.cat((f[:, crop:], torch.zeros_like(f[:, :crop - tp])), 1) for f in full)
    else:
        acc = _conv64(x, w, stride, pad, out_sp)
        S = _conv64(x.abs(), w.abs(), stride, pad, out_sp)
    if delta is not None:
        acc = acc + delta
    if os is not None:
        osv = os.clone()
        if wrong == "oscale of clip 0 used for clip 1":
            osv[1:] = osv[0]
        osb = osv[:, None, None, None, :]
        S = S * os.abs()[:, None, None, None, :]
    gam = _gamma(K, C_KERN[kern])
    if os is not None and wrong == "oscale applied after the bias":
        z = (acc + b) * osb
    elif os is not None:
        z = acc * osb + b
    else:
        z = acc + b
    if wrong == "bias dropped":
        z = z - b
    if exact:                     # with oscale the product and the bias add still round: 3 u (S |os| + |b|) covers both
        e = torch.zeros_like(S) if os is None else 3 * U * (S + b.abs())
    else:
        e = gam * S + 3 * U * (S + b.abs())
    if wrong == "bias added after the activation":
        v = ACT64[act](z - b) + b
    else:
        v = ACT64[act](z)
    e = SLOPE[act] * e + _act_err(act, z, v, kern)
    ref = v
    if r is not None:
        t = v + r
        e = e + U * t.abs()
        ref = t
        if mode == 2:
            ref = v * RS + r if wrong == "scaled-residual factor applied before the residual add" else t * RS
            if kern == "simt":    # rounded to the output dtype, then scaled and rounded again
                e = RS * (0.5 * _ulp(t.abs() + e, dtype) + e) + 2 * U * ref.abs()
            else:
                e = RS * e + 2 * U * ref.abs()
    swap = wrong == "shuffle phases swapped"
    ref, e = _shuffle(ref, shuffle, swap), _shuffle(e, shuffle)
    if tp is not None:
        ref, e = ref.permute(0, 4, 1, 2, 3), e.permute(0, 4, 1, 2, 3)
    return ref, e


def _forward64(c, x, w, b, os, r, wrong=None):
    """forward64 of case c."""
    pad, out_sp = _geometry(c)
    K = 12 * c.ci if c.kern == "down" else math.prod(c.k) * c.ci      # the packed down-space GEMM: 6 taps x 2 Ci
    return forward64(x, w, b, os, r, kern=c.kern, stride=c.stride, pad=pad, out_sp=out_sp, K=K, act=c.act, mode=c.mode,
                     shuffle=c.shuffle, tp=c.tp, tshift=c.tshift, dtype=DT[c.dt], wrong=wrong)


def _wrongs(c):
    """The defects case c's bound must reject."""
    out = ["bias dropped"]
    if c.act != NONE:
        out.append("bias added after the activation")
    if c.oscale:
        out += ["oscale applied after the bias"] + (["oscale of clip 0 used for clip 1"] if c.shape[0] > 1 else [])
    if c.mode == 2:
        out.append("scaled-residual factor applied before the residual add")
    if c.shuffle != SHUFFLE_NONE:
        out.append("shuffle phases swapped")
    if 2 in c.stride:
        out.append("pad at the back")
    if c.tp is not None:
        out.append("cropped one frame late")
    if c.tshift:
        out.append("token shift split at floor(Ci / 2)")
    return out


# ------------------------------------------------------------------------------------------------------------------
# families 1 - 3 and 5: one Engine.conv call against float64
# ------------------------------------------------------------------------------------------------------------------
CONV_CASES = [
    # ---- 1. slab EPI_PLAIN: every activation, bn 32 / 64 / 128, mw 1 / 2 / 4, ragged planes, T = 1, 64-byte rows ----
    case("slab_plain_none_bn64_mw2_24x20", "slab", shape=(2, 3, 24, 20), plan=(2, 64, 1, 2)),
    case("slab_plain_elu_bn128_mw1_20x12", "slab", co=128, shape=(1, 2, 20, 12), act=ELU, plan=(1, 128, 1, 3)),
    case("slab_plain_silu_bn32_k133_T1", "slab", co=32, k=K133, shape=(2, 1, 12, 36), act=SILU, plan=(2, 32, 1, 3)),
    case("slab_plain_leaky_ci32_kw1", "slab", ci=32, k=(3, 3, 1), shape=(2, 3, 18, 20), act=LEAKY, plan=(2, 64, 1, 3)),
    case("slab_plain_relu_co96_bn32x3", "slab", co=96, k=K111, shape=(1, 2, 17, 40), act=RELU, plan=(4, 32, 3, 2)),
    case("slab_plain_wide_co1376_ragged128", "slab", co=1376, k=K111, shape=(1, 1, 9, 10), plan=(1, 128, 11, 3)),
    case("slab_plain_elu_oscale_b2", "slab", shape=(2, 2, 20, 12), act=ELU, oscale=True, plan=(2, 64, 1, 2)),
    case("slab_plain_silu_oscale_bn128", "slab", co=128, k=K133, shape=(2, 1, 12, 20), act=SILU, oscale=True,
         plan=(1, 128, 1, 3)),
    # ---- EPI_PLAIN_RES ----
    case("slab_res_elu", "slab", shape=(2, 2, 20, 12), act=ELU, res=True, plan=(2, 64, 1, 2)),
    case("slab_res_mode2_leaky_c128", "slab", co=128, k=K133, shape=(2, 1, 24, 20), act=LEAKY, res=True, mode=2,
         plan=(1, 128, 1, 3)),
    case("slab_res_co96_bn32_mw4", "slab", co=96, k=K111, shape=(1, 2, 9, 36), act=SILU, res=True, plan=(4, 32, 3, 2)),
    case("slab_res_oscale_b2", "slab", k=K133, shape=(2, 2, 12, 20), act=ELU, res=True, oscale=True, plan=(2, 64, 1, 2)),
    # ---- EPI_RAGGED ----
    case("slab_ragged_co3", "slab", co=3, shape=(2, 3, 20, 12), plan=(2, 32, 1, 3)),
    case("slab_ragged_co3_oscale_silu", "slab", co=3, shape=(2, 2, 12, 20), act=SILU, oscale=True, plan=(2, 32, 1, 3)),
    case("slab_ragged_co13_elu", "slab", co=13, shape=(1, 2, 18, 24), act=ELU, plan=(2, 32, 1, 3)),
    case("slab_ragged_co13_oscale", "slab", co=13, k=K133, shape=(2, 1, 18, 24), act=ELU, oscale=True, plan=(2, 32, 1, 3)),
    case("slab_conv_out_cf_tp0", "slab", co=3, shape=(2, 3, 12, 20), tp=0, plan=(2, 32, 1, 3)),
    case("slab_conv_out_cf_tp1", "slab", co=3, shape=(2, 4, 12, 20), tp=1, plan=(2, 32, 1, 3)),
    case("slab_conv_out_cf_tp3", "slab", co=3, shape=(1, 6, 20, 12), tp=3, plan=(2, 32, 1, 3)),
    # ---- EPI_SHUFFLE_ST (Cy % 32 == 0) and EPI_SHUFFLE (Cy 16 / 24; time Cy 16) ----
    case("slab_shuffle_st_space_cy32", "slab", co=128, k=K111, shape=(2, 2, 12, 20), act=SILU, shuffle=SHUFFLE_SPACE,
         plan=(1, 128, 1, 3)),
    case("slab_shuffle_st_time_cy32", "slab", co=64, k=K111, shape=(1, 3, 20, 12), act=SILU, shuffle=SHUFFLE_TIME,
         plan=(2, 64, 1, 3)),
    case("slab_shuffle_space_cy16", "slab", co=64, k=K111, shape=(1, 2, 12, 20), act=SILU, shuffle=SHUFFLE_SPACE,
         plan=(2, 64, 1, 3)),
    case("slab_shuffle_space_cy24", "slab", co=96, k=K111, shape=(2, 1, 12, 20), act=SILU, shuffle=SHUFFLE_SPACE,
         plan=(4, 32, 3, 2)),
    case("slab_shuffle_time_cy16", "slab", co=32, k=K111, shape=(1, 3, 12, 20), act=SILU, shuffle=SHUFFLE_TIME,
         plan=(4, 32, 1, 2)),
    # ---- time-strided slab (TimeDownsample2x) ----
    case("slab_time_down_T5", "slab", k=(3, 1, 1), stride=(2, 1, 1), pad=(2, 0, 0), shape=(2, 5, 12, 20),
         plan=(2, 64, 1, 3)),
    case("slab_time_down_T2_ci128_co64", "slab", ci=128, k=(3, 1, 1), stride=(2, 1, 1), pad=(2, 0, 0),
         shape=(2, 2, 12, 20), plan=(2, 64, 1, 3)),
    case("slab_time_down_T7_ci64_co128", "slab", co=128, k=(3, 1, 1), stride=(2, 1, 1), pad=(2, 0, 0),
         shape=(1, 7, 20, 12), plan=(1, 128, 1, 3)),
    # ---- 2. down-space slab, and an odd plane on the tap-wise kernel ----
    case("down_space_c64_co128", "down", co=128, k=K133, stride=(1, 2, 2), pad=(0, 1, 1), shape=(2, 2, 40, 36), down=True),
    case("down_space_c128_co64", "down", ci=128, co=64, k=K133, stride=(1, 2, 2), pad=(0, 1, 1), shape=(1, 2, 24, 52),
         down=True),
    case("down_space_c64_co96_bn32", "down", co=96, k=K133, stride=(1, 2, 2), pad=(0, 1, 1), shape=(2, 1, 26, 44), down=True),
    case("down_space_odd_h_falls_back_to_tap", "tap", k=K133, stride=(1, 2, 2), pad=(0, 1, 1), shape=(1, 2, 23, 20),
         down=True),
    case("down_space_odd_w_falls_back_to_tap", "tap", ci=128, co=64, k=K133, stride=(1, 2, 2), pad=(0, 1, 1),
         shape=(1, 1, 16, 21), down=True),
    # ---- 3. tap-wise kernel ----
    case("tap_bk16_ci16_elu", "tap", ci=16, co=32, shape=(2, 3, 12, 20), act=ELU),
    case("tap_bk16_ci48_bn64", "tap", variant="tap", ci=48, co=64, shape=(1, 2, 12, 20), act=SILU),
    case("tap_bk32_ci32_bn128", "tap", variant="tap", ci=32, co=128, shape=(1, 2, 12, 20), act=LEAKY),
    case("tap_bk64_co96_ragged_n", "tap", variant="tap", co=96, shape=(1, 2, 12, 20), act=RELU),
    case("tap_bk64_co160_two_n_tiles", "tap", variant="tap", co=160, k=K133, shape=(2, 1, 12, 20), act=ELU),
    case("tap_box_wide_w130", "tap", variant="tap", co=32, k=K133, shape=(1, 2, 3, 130), act=ELU),
    case("tap_box_small_plane_T5", "tap", variant="tap", co=32, shape=(2, 5, 4, 4), act=ELU),
    case("tap_box_w5", "tap", variant="tap", co=32, shape=(1, 3, 6, 5), act=SILU),
    case("tap_k111_loop_shorter_than_ring", "tap", variant="tap", co=64, k=K111, shape=(2, 3, 12, 20), act=ELU),
    case("tap_stride_122_odd", "tap", variant="tap", co=64, k=K133, stride=(1, 2, 2), pad=(0, 1, 1), shape=(1, 2, 13, 11),
         act=ELU),
    case("tap_stride_211_odd_T7", "tap", variant="tap", ci=32, co=64, k=(3, 1, 1), stride=(2, 1, 1), pad=(2, 0, 0),
         shape=(2, 7, 5, 9)),
    case("tap_ragged_co3_silu", "tap", variant="tap", co=3, shape=(2, 2, 12, 20), act=SILU),
    case("tap_ragged_co13_oscale", "tap", variant="tap", co=13, shape=(2, 2, 12, 20), act=ELU, oscale=True),
    case("tap_res_elu", "tap", variant="tap", co=64, shape=(2, 2, 12, 20), act=ELU, res=True),
    case("tap_res_mode2_leaky", "tap", variant="tap", co=128, k=K133, shape=(2, 1, 12, 20), act=LEAKY, res=True, mode=2),
    case("tap_oscale_b2_silu", "tap", variant="tap", co=64, shape=(2, 2, 12, 20), act=SILU, oscale=True),
    case("tap_shuffle_space_cy24_ragged", "tap", variant="tap", co=96, k=K111, shape=(2, 2, 12, 20), act=SILU,
         shuffle=SHUFFLE_SPACE),
    case("tap_shuffle_space_cy16", "tap", variant="tap", co=64, k=K111, shape=(1, 2, 12, 20), act=SILU,
         shuffle=SHUFFLE_SPACE),
    case("tap_shuffle_space_cy8_bn32", "tap", variant="tap", co=32, k=K111, shape=(2, 1, 12, 20), act=SILU,
         shuffle=SHUFFLE_SPACE),
    case("tap_shuffle_time_cy24", "tap", co=48, k=K111, shape=(1, 3, 12, 20), act=SILU, shuffle=SHUFFLE_TIME),
    # ---- 5. CUDA-core conv, bf16 and fp32 ----
    case("simt_bf16_ci3_co70_oscale_elu", "simt", variant="simt", ci=3, co=70, shape=(2, 3, 9, 10), act=ELU, oscale=True),
    case("simt_f32_ci5_co67_silu", "simt", dt="f32", ci=5, co=67, k=K133, shape=(2, 2, 9, 11), act=SILU),
    case("simt_bf16_ci48_res_leaky", "simt", variant="simt", ci=48, co=48, shape=(1, 2, 9, 10), act=LEAKY, res=True),
    case("simt_f32_ci48_relu_oscale", "simt", dt="f32", ci=48, co=40, shape=(2, 2, 7, 9), act=RELU, oscale=True),
    case("simt_f32_token_shift_ci5", "simt", dt="f32", ci=5, co=16, k=K111, shape=(2, 3, 5, 6), tshift=True),
    case("simt_bf16_token_shift_ci7_T1", "simt", variant="simt", ci=7, co=16, k=K111, shape=(2, 1, 5, 6), tshift=True,
         act=ELU),
    case("simt_bf16_token_shift_ci7", "simt", variant="simt", ci=7, co=24, k=K333, shape=(1, 4, 5, 6), tshift=True),
    case("simt_bf16_shuffle_space", "simt", variant="simt", ci=48, co=32, k=K111, shape=(1, 2, 5, 7), act=SILU,
         shuffle=SHUFFLE_SPACE),
    case("simt_f32_shuffle_space", "simt", dt="f32", ci=5, co=12, k=K111, shape=(2, 2, 5, 7), act=SILU,
         shuffle=SHUFFLE_SPACE),
    case("simt_f32_shuffle_time", "simt", dt="f32", ci=5, co=10, k=K111, shape=(1, 3, 5, 7), act=SILU,
         shuffle=SHUFFLE_TIME),
    case("simt_bf16_stride_122_odd", "simt", variant="simt", ci=5, co=20, k=K133, stride=(1, 2, 2), pad=(0, 1, 1),
         shape=(2, 2, 13, 11)),
    case("simt_f32_stride_211_odd", "simt", dt="f32", ci=48, co=24, k=(3, 1, 1), stride=(2, 1, 1), pad=(2, 0, 0),
         shape=(2, 7, 5, 9)),
    case("simt_bf16_mode2_two_roundings", "simt", variant="simt", ci=48, co=40, k=K133, shape=(2, 1, 9, 10), act=LEAKY,
         res=True, mode=2),
    case("simt_f32_mode2", "simt", dt="f32", ci=3, co=40, k=K133, shape=(2, 1, 9, 10), act=LEAKY, res=True, mode=2),
]


@pytest.mark.parametrize("c", CONV_CASES)
def test_conv_forward_vs_float64(guarded, c):
    dtype = DT[c.dt]
    eng = _engine(dtype, c.variant)
    guarded(eng)
    gen = _gen(c.name)
    B, T, H, W = c.shape
    w = _bfrand((c.co, c.ci, *c.k), gen, (c.ci * math.prod(c.k)) ** -0.5)
    b = _bfrand(c.co, gen, 0.5)
    x = _bfrand((B, T, H, W, c.ci), gen)
    pad, out_sp = _geometry(c)
    q = 4 if c.shuffle == SHUFFLE_SPACE else 2 if c.shuffle == SHUFFLE_TIME else 1
    if c.down:                    # SpatialDownsample2x: a Conv2d weight, packed for the down-space slab
        w2 = w[:, :, 0]
        pk = pack_conv(w2.float(), b.float(), dtype)
        if dtype == torch.bfloat16:
            pack_conv_down_space(pk, w2.float())
    else:
        pk = pack_conv(w.float(), b.float(), dtype, k=c.k, shuffle_q=q)
    pk.epi_mode = c.mode
    To, Ho, Wo = out_sp
    y_shape = {SHUFFLE_NONE: (B, To, Ho, Wo, c.co), SHUFFLE_SPACE: (B, To, 2 * Ho, 2 * Wo, c.co // 4),
               SHUFFLE_TIME: (B, 2 * To, Ho, Wo, c.co // 2)}[c.shuffle]
    r = _bfrand(y_shape, gen) if c.res else None
    os = None
    if c.oscale:                  # Conv3DMod demodulation factors, a different set per clip
        os = (torch.rand((B, c.co), generator=gen, device="cuda", dtype=torch.float64) * 1.5 + 0.25).float().double()
        os[1:] *= 2.5
    kw = dict(stride=c.stride, pad=pad, out_spatial=out_sp, act=c.act, shuffle=c.shuffle, token_shift=c.tshift,
              out_cf=c.tp is not None)
    if r is not None:
        kw["res"] = r.to(dtype).contiguous()
    if os is not None:
        kw["oscale"] = os.float().contiguous()
    kind, y = _ran(eng, lambda: eng.conv(x.to(dtype).contiguous(), pk, **kw))
    assert kind == c.kern, f"{c.name}: expected the {c.kern} kernel, ran {kind}"
    if kind == "slab":
        got = _slab_plan(x.shape, pk, c.stride, pad, out_sp, c.shuffle, c.res, c.oscale, c.tp is not None)
        assert got == c.plan, f"{c.name}: slab plan (mw, bn, n_tiles_n, slab_stages) {got}, the case claims {c.plan}"
        rec = eng.conv_log[-1]
        assert (rec["act"], rec["shuffle"], rec["res"], rec["epi_mode"]) == (c.act, c.shuffle, c.res, c.mode)
    assert y.dtype == dtype and y.shape == ((B, c.co, *out_sp) if c.tp is not None else y_shape)
    ref, acc = _forward64(c, x, w, b.double(), os, r)
    _check(y, ref, dtype, acc, c.name)
    for wrong in _wrongs(c):
        wref, _ = _forward64(c, x, w, b.double(), os, r, wrong)
        _rejects(y, wref, dtype, acc, f"{c.name}: {wrong}")


# ------------------------------------------------------------------------------------------------------------------
# EPI_GEGLU: fc1 + GEGLU fused (pack_ff and hand-packed widths)
# ------------------------------------------------------------------------------------------------------------------
def _pack_geglu(w1, b1):
    """fc1 (2I, C) rows re-paired as pack_ff does, [8 x rows, their 8 gate rows] per 16, WITHOUT padding I (I % 8 == 0):
    the C ABI's GEGLU epilogue at widths pack_ff never produces."""
    two_i, C_ = w1.shape
    I = two_i // 2
    wp = torch.stack((w1[:I].reshape(I // 8, 8, C_), w1[I:].reshape(I // 8, 8, C_)), 1).reshape(two_i, C_)
    bp = torch.stack((b1[:I].reshape(I // 8, 8), b1[I:].reshape(I // 8, 8)), 1).reshape(two_i)
    return ConvPack(w=None, bias=None, k=(1, 1, 1), Ci=C_, Co=two_i, w_tc=wp.to(torch.bfloat16).contiguous(),
                    bias_tc=bp.float().contiguous(), Ci_tc=C_, Co_tc=two_i, epi_mode=1, k_tc=(1, 1, 1))


GEGLU_CASES = [
    # name, C, I, packing, variant, (B, T, H, W), kernel, slab plan.  pack_ff pads I to a multiple of 64 (Co 128 k).
    ("geglu_pack_ff_c64", 64, 170, "ff", "auto", (1, 2, 12, 20), "slab", (1, 128, 3, 3)),
    ("geglu_pack_ff_c256", 256, 682, "ff", "auto", (1, 1, 9, 10), "slab", (1, 128, 11, 3)),
    ("geglu_pack_ff_c512", 512, 1365, "ff", "auto", (1, 1, 8, 12), "slab", (1, 128, 22, 3)),
    ("geglu_hand_co192_bn64", 64, 96, "hand", "auto", (2, 1, 12, 20), "slab", (2, 64, 3, 3)),
    ("geglu_hand_co2752_ragged128", 512, 1376, "hand", "auto", (1, 1, 8, 12), "slab", (1, 128, 22, 3)),
    ("geglu_tap_pack_ff_c64", 64, 170, "ff", "tap", (1, 2, 12, 20), "tap", None),
    ("geglu_tap_hand_co96", 48, 48, "hand", "tap", (1, 2, 12, 20), "tap", None),
    ("geglu_tap_hand_co32_bn32", 32, 16, "hand", "tap", (2, 1, 12, 20), "tap", None),
    ("geglu_tap_hand_co64_bn64", 64, 32, "hand", "tap", (1, 2, 12, 20), "tap", None),
]


@pytest.mark.parametrize("name,C_,I,packing,variant,shape,kern,plan", GEGLU_CASES, ids=[c[0] for c in GEGLU_CASES])
def test_geglu_epilogue_vs_float64(guarded, name, C_, I, packing, variant, shape, kern, plan):
    eng = _engine(torch.bfloat16, variant)
    guarded(eng)
    gen = _gen(name)
    B, T, H, W = shape
    w1 = _bfrand((2 * I, C_), gen, C_ ** -0.5)
    b1 = _bfrand(2 * I, gen, 0.5)
    x = _bfrand((B, T, H, W, C_), gen)
    if packing == "ff":
        w2 = _bfrand((C_, I), gen, I ** -0.5)
        pk, _ = pack_ff(w1.float()[..., None, None, None], b1.float(), w2.float()[..., None, None, None],
                        torch.zeros(C_, device="cuda"), torch.bfloat16)
    else:
        pk = _pack_geglu(w1.float(), b1.float())
    kind, y = _ran(eng, lambda: eng.conv(x.to(torch.bfloat16), pk))
    assert kind == kern, f"{name}: expected the {kern} kernel, ran {kind}"
    if kind == "slab":
        assert _slab_plan(x.shape, pk, (1, 1, 1), (0, 0, 0), (T, H, W), 0, False, False, False) == plan
        assert eng.conv_log[-1]["geglu"]
    Ip = pk.Co_tc // 2
    assert y.shape == (B, T, H, W, Ip)
    if Ip > I:                    # the hidden channels pack_ff pads in are exactly zero: gelu(0) * 0
        assert torch.equal(y[..., I:].float(), torch.zeros_like(y[..., I:].float())), f"{name}: padded channels"
    ref, acc, (xv, gt) = geglu64(x, w1, b1, kind)
    out = y[..., :I]
    _check(out, ref, torch.bfloat16, acc, name)
    _rejects(out, F.gelu(xv) * gt, torch.bfloat16, acc, f"{name}: x and gate halves swapped")
    _rejects(out, (F.gelu(gt - b1[I:]) + b1[I:]) * xv, torch.bfloat16, acc, f"{name}: gate bias added after the GELU")


def geglu64(x, w1, b1, kern, exact=False):
    """float64 fc1 + GEGLU of x (..., C) with fc1 (2I, C) in the reference's row order: (reference, allowance, (x half,
    gate half)).  `exact`: fc1's accumulation and bias add are exact (dyadic operands)."""
    I = w1.shape[0] // 2
    h = x @ w1.T + b1
    S = x.abs() @ w1.abs().T
    e = torch.zeros_like(S) if exact else _gamma(w1.shape[1], C_KERN[kern]) * S + 3 * U * (S + b1.abs())
    xv, gt, ex, eg = h[..., :I], h[..., I:], e[..., :I], e[..., I:]
    ref = F.gelu(gt) * xv
    acc = xv.abs() * (_gelu_err(gt) + GELU_SLOPE * eg) + F.gelu(gt).abs() * ex + U * ref.abs()
    return ref, acc, (xv, gt)


# ------------------------------------------------------------------------------------------------------------------
# 4. kw-packed conv_in
# ------------------------------------------------------------------------------------------------------------------
KWPACK_CASES = [
    # name, variant, (B, T, H, W), time padding frames, kernel, slab plan
    ("kwpack_slab_T5_20x20", "auto", (2, 5, 20, 20), 0, "slab", (2, 64, 1, 2)),
    ("kwpack_slab_T1_tpad3", "auto", (2, 1, 12, 20), 3, "slab", (2, 64, 1, 2)),
    ("kwpack_tap_T5_20x20", "tap", (2, 5, 20, 20), 0, "tap", None),
    ("kwpack_tap_T1_tpad3", "tap", (2, 1, 12, 20), 3, "tap", None),
]


@pytest.mark.parametrize("name,variant,shape,t_pad,kern,plan", KWPACK_CASES, ids=[c[0] for c in KWPACK_CASES])
def test_kwpack_conv_in_vs_float64(guarded, name, variant, shape, t_pad, kern, plan):
    """The channels-first video through mv2_ingest_kwpack and the 49-tap conv against the float64 7x7x7 causal conv
    (pad (6, 3, 3) after t_pad leading zero frames), so the packing is checked together with the kernel."""
    eng = _engine(torch.bfloat16, variant)
    guarded(eng)
    gen = _gen(name)
    B, T, H, W = shape
    Co = 64
    w = _bfrand((Co, 3, 7, 7, 7), gen, (3 * 343) ** -0.5)
    b = _bfrand(Co, gen, 0.5)
    video = _bfrand((B, 3, T, H, W), gen)
    pin = pack_conv_in_kwpack(w.float(), b.float())
    x = eng.ingest_kwpack(video.to(torch.bfloat16), t_pad, pin)
    assert x.shape == (B, T + t_pad, H, W, 32)
    kind, y = _ran(eng, lambda: eng.conv(x, pin, pad=(6, 3, 0), act=LEAKY))
    assert kind == kern, f"{name}: expected the {kern} kernel, ran {kind}"
    if kind == "slab":
        assert _slab_plan(x.shape, pin, (1, 1, 1), (6, 3, 0), (T + t_pad, H, W), 0, False, False, False) == plan
    v = F.pad(video.permute(0, 2, 3, 4, 1), (0, 0, 0, 0, 0, 0, t_pad, 0))
    out_sp = (T + t_pad, H, W)
    z = _conv64(v, w, (1, 1, 1), (6, 3, 3), out_sp) + b
    S = _conv64(v.abs(), w.abs(), (1, 1, 1), (6, 3, 3), out_sp)
    acc = _gamma(7 * 7 * 32, C_KERN[kind]) * S + 3 * U * (S + b.abs())
    ref = F.leaky_relu(z, 0.1)
    _check(y, ref, torch.bfloat16, acc, name)
    _rejects(y, F.leaky_relu(_conv64(v, w.flip(4), (1, 1, 1), (6, 3, 3), out_sp) + b, 0.1), torch.bfloat16, acc,
             f"{name}: the kw taps mirrored")
    _rejects(y, F.leaky_relu(_conv64(v, w, (1, 1, 1), (0, 3, 3), out_sp) + b, 0.1), torch.bfloat16, acc,
             f"{name}: time pad at the back")
    _rejects(y, F.leaky_relu(z - b, 0.1) + b, torch.bfloat16, acc, f"{name}: bias added after the activation")


# ------------------------------------------------------------------------------------------------------------------
# 6. fused ResidualUnit: y and the SqueezeExcite gates
# ------------------------------------------------------------------------------------------------------------------
RU_CASES = [
    # name, C, (B, T, H, W), (mw, bn, n_tiles_n) of its 3x3x3 conv's slab plan (the fused kernel sets its own stages).  H % 16 = 4 / 8 / 12 leaves whole 32-position quarters of the
    # last row tile outside the frame; W is not a multiple of 8 mw; the last case has more tiles than SMs.
    ("ru_c64_h20_w24_b2", 64, (2, 2, 20, 24), (2, 64, 1)),
    ("ru_c128_h24_w20_T1", 128, (1, 1, 24, 20), (1, 128, 1)),
    ("ru_c64_h28_w20_T1_b2", 64, (2, 1, 28, 20), (2, 64, 1)),
    ("ru_c128_h12_w12_b2", 128, (2, 3, 12, 12), (1, 128, 1)),
    ("ru_c64_200_tiles", 64, (2, 5, 60, 72), (2, 64, 1)),
]
RU_HD = 32


def ru_y64(x, w3, b3, w1, b1, exact=False, delta=None):
    """float64 y = ELU(conv1(round_bf16(ELU(conv3 x + b3))) + b1) of the fused ResidualUnit (module docstring): (y,
    allowance, bf16-rounded h).  x (B,T,H,W,C), w3 (C,C,kt,kh,kw), w1 (C,C,1,1,1).  `exact`: conv3's accumulation and bias
    add are exact (dyadic operands); `delta` is added to conv3's accumulators."""
    B, T, H, W, C_ = x.shape
    kt, kh, kw = w3.shape[2:]
    K3 = kt * kh * kw * C_
    z3 = _conv64(x, w3, (1, 1, 1), (kt - 1, kh // 2, kw // 2), (T, H, W))
    if delta is not None:
        z3 = z3 + delta
    z3 = z3 + b3
    h64 = F.elu(z3)
    eh = _act_err(ELU, z3, h64, "slab")
    if not exact:
        S3 = _conv64(x.abs(), w3.abs(), (1, 1, 1), (kt - 1, kh // 2, kw // 2), (T, H, W))
        eh = eh + _gamma(K3, 2) * S3 + 3 * U * (S3 + b3.abs())
        del S3
    lo, hi = (v.to(torch.bfloat16).double() for v in (h64 - eh, h64 + eh))
    hb = h64.to(torch.bfloat16).double()
    del h64, eh, z3
    either = torch.where(lo != hi, _ulp(torch.maximum(lo.abs(), hi.abs()), torch.bfloat16), torch.zeros_like(hb))
    del lo, hi
    w1m = w1[:, :, 0, 0, 0]
    z1 = hb @ w1m.T + b1
    S1 = (hb.abs() + either) @ w1m.abs().T
    y_ref = F.elu(z1)
    ey = _gamma(C_, 2) * S1 + 3 * U * (S1 + b1.abs()) + either @ w1m.abs().T + _act_err(ELU, z1, y_ref, "slab")
    return y_ref, ey, hb


def _ru_targets(H, W):
    """Impulse positions per frame: the last (ragged) row's last column, elsewhere on the last row and on the last column,
    and next to a quarter boundary (rows 3 / 4 of a row tile)."""
    return [(H - 1, W - 1), (H - 1, W // 3), (H // 3, W - 1), (4, 5)]


@pytest.mark.parametrize("name,C_,shape,plan", RU_CASES, ids=[c[0] for c in RU_CASES])
def test_fused_residual_unit_vs_float64(guarded, name, C_, shape, plan):
    eng = _engine(torch.bfloat16, "auto")
    guard = guarded(eng)
    gen = _gen(name)
    B, T, H, W = shape
    w3 = _bfrand((C_, C_, 3, 3, 3), gen, (27 * C_) ** -0.5)
    b3 = _bfrand(C_, gen, 0.5)
    w1 = _bfrand((C_, C_, 1, 1, 1), gen, C_ ** -0.5)
    b1 = _bfrand(C_, gen, 0.5)
    # a sparse impulse input, one channel vector per position in every frame (so one se_wk can favour the same position
    # in every frame): the positions the pool must not lose dominate their frame's softmax
    x = torch.zeros((B, T, H, W, C_), device="cuda", dtype=torch.float64)
    for (h, w_) in _ru_targets(H, W):
        x[:, :, h, w_] = _bfrand(C_, gen, 3.0)
    x[1:] *= 2                                                      # clip 1 scaled
    y_ref, ey, hb = ru_y64(x, w3, b3, w1, b1)
    w1m = w1[:, :, 0, 0, 0]
    # se_wk along the corner impulse's response in y, scaled until the last row and the last column each carry at least
    # 10% of every frame's softmax weight
    y_bg = y_ref[0, 0, 0, 0]                                       # no impulse reaches (0, 0): the constant background
    d = (y_ref[:, :, H - 1, W - 1] - y_bg).reshape(-1, C_).sum(0)
    d = d / d.norm()
    last_row = [(H - 1) * W + w_ for w_ in range(W)]
    last_col = [h * W + W - 1 for h in range(H)]
    for scale in (1.25 ** i for i in range(30)):
        wk = (d * scale).float().double()
        p_ = (y_ref.reshape(B * T, H * W, C_) @ wk).softmax(-1)
        if min(p_[:, last_row].sum(-1).min().item(), p_[:, last_col].sum(-1).min().item()) >= 0.1:
            break
    assert p_[:, last_row].sum(-1).min().item() >= 0.1, f"{name}: the last row carries < 10% of a frame's softmax"
    assert p_[:, last_col].sum(-1).min().item() >= 0.1, f"{name}: the last column carries < 10% of a frame's softmax"
    prm = dict(wk=wk, bk=0.25, w1=_bfrand((RU_HD, C_), gen, 2 * C_ ** -0.5), b1=_bfrand(RU_HD, gen, 0.1),
               w2=_bfrand((C_, RU_HD), gen, 2 * RU_HD ** -0.5), b2=_bfrand(C_, gen, 0.1))
    p = dict(conv3=pack_conv(w3.float(), b3.float(), torch.bfloat16), conv1=pack_conv(w1.float(), b1.float(), torch.bfloat16),
             wk=prm["wk"].float().contiguous(), bk=prm["bk"], w1=prm["w1"].float().contiguous(),
             b1=prm["b1"].float().contiguous(), w2=prm["w2"].float().contiguous(), b2=prm["b2"].float().contiguous(),
             hidden=RU_HD)
    kind, _ = _ran(eng, lambda: eng.residual_unit(x.to(torch.bfloat16), p))
    assert kind == "ru", f"{name}: expected the fused ResidualUnit kernel, ran {kind}"
    assert eng.conv_log[-1].get("fused_ru")
    pk3 = p["conv3"]
    assert _slab_plan(x.shape, pk3, (1, 1, 1), (2, 1, 1), (T, H, W), 0, False, False, False)[:3] == plan
    y, gates = guard.allocs[0][0][HEAD:HEAD + y_ref.numel()].view(y_ref.shape), guard.allocs[2][0]
    gates = gates[HEAD:HEAD + B * T * C_].view(B * T, C_)
    # y
    _check(y, y_ref, torch.bfloat16, ey, f"{name}: y")
    _rejects(y, F.elu(hb @ w1m.T) + b1, torch.bfloat16, ey, f"{name}: y with b1 added after the ELU")
    # gates, from the kernel's own bf16 y
    y_own = y.double().reshape(B * T, H * W, C_)
    g_ref = _se_gates64(y_own, prm)
    err = (gates.double() - g_ref).abs().max().item()
    assert err <= GATE_TOL, f"{name}: gates vs float64 {err:.3g}"
    for drop, what in ((last_row, "without the frame's last ragged row"), (last_col, "without its last column")):
        wrong = _se_gates64(y_own, prm, drop=torch.tensor(drop, device="cuda"))
        assert (gates.double() - wrong).abs().max().item() > GATE_TOL, f"{name}: the gate bound accepts gates {what}"
