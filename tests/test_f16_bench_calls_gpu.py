"""Every conv-path kernel call of the benchmark's tokenize + decode, in fp16 (``model.half()``), checked one call at a time
against float64 at the benchmark's own shapes: tests/test_bench_calls_gpu.py's three parts (real data call by call, the
exact replay on a dyadic grid with its pipeline defects, the launch mode) run unchanged on an fp16 model.

What changes with the dtype is the storage rounding, so the bounds are the bf16 ones with fp16's unit: every stored value
may be off by half an fp16 ulp (11 significant bits) instead of half a bf16 ulp, and the fused ResidualUnit's 1x1x1 GEMM
reads h rounded to fp16.  The replay grid (x, residual and video in {-8..8} / 2^2, weights in {-8..8} / 2^6, biases in
{-64..64} / 2^8, oscale in {1..8} / 2^3) is exact in fp16 as it is in bf16 (test_replay_grid_is_exact_in_fp16), so the
replay still leaves only the epilogue's roundings to allow for."""
import functools

import pytest
import torch
import torch.nn.functional as F

import synth_data
import tests.test_bench_calls_gpu as BC
import tests.test_conv_forward_gpu as CF
import tests.test_simt_ops_gpu as SO
from bench import WORKLOADS
from magvit2_pytorch_b200 import VideoTokenizer

pytestmark = pytest.mark.gpu

H = torch.float16
_EAGER = {}


def _ulp16(v, dtype):
    """ulp of |v| in `dtype`, elementwise (float64), 0 where v == 0.  fp16: 11 significant bits, and below 2^-14 the
    subnormals' fixed spacing 2^-24 (bf16 and fp32 reach no subnormal value here)."""
    p = 11 if dtype == torch.float16 else (8 if dtype == torch.bfloat16 else 24)
    _, e = torch.frexp(v.abs())
    ex = e - p
    if dtype == torch.float16:
        ex = torch.clamp(ex, min=-24)
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), ex))


def _ru_y64_f16(x, w3, b3, w1, b1, exact=False, delta=None):
    """CF.ru_y64 with h rounded to fp16, the fused ResidualUnit's rounding point in an fp16 model."""
    B, T, Hh, W, C_ = x.shape
    kt, kh, kw = w3.shape[2:]
    K3 = kt * kh * kw * C_
    z3 = CF._conv64(x, w3, (1, 1, 1), (kt - 1, kh // 2, kw // 2), (T, Hh, W))
    if delta is not None:
        z3 = z3 + delta
    z3 = z3 + b3
    h64 = F.elu(z3)
    eh = CF._act_err(CF.ELU, z3, h64, "slab")
    if not exact:
        S3 = CF._conv64(x.abs(), w3.abs(), (1, 1, 1), (kt - 1, kh // 2, kw // 2), (T, Hh, W))
        eh = eh + CF._gamma(K3, 2) * S3 + 3 * CF.U * (S3 + b3.abs())
    lo, hi = (v.to(H).double() for v in (h64 - eh, h64 + eh))
    hb = h64.to(H).double()
    either = torch.where(lo != hi, _ulp16(torch.maximum(lo.abs(), hi.abs()), H), torch.zeros_like(hb))
    w1m = w1[:, :, 0, 0, 0]
    z1 = hb @ w1m.T + b1
    S1 = (hb.abs() + either) @ w1m.abs().T
    y_ref = F.elu(z1)
    ey = CF._gamma(C_, 2) * S1 + 3 * CF.U * (S1 + b1.abs()) + either @ w1m.abs().T + CF._act_err(CF.ELU, z1, y_ref, "slab")
    return y_ref, ey, hb


def _workload_f16(name):
    wl = WORKLOADS[name]
    torch.manual_seed(0)
    model = VideoTokenizer(**wl["kw"])
    synth_data.fill_state_dict_(model, 0)
    model = model.cuda().half().eval()
    clips = wl["clips"] if name == "readme" else 1
    return model, clips, wl["size"]


@pytest.fixture
def f16(monkeypatch):
    monkeypatch.setattr(BC, "BF", H)
    monkeypatch.setattr(BC, "_workload", _workload_f16)
    monkeypatch.setattr(BC, "ru_y64", _ru_y64_f16)
    # the replay packs conv_in itself: in the model's dtype (the packer's default is bf16)
    monkeypatch.setattr(BC, "pack_conv_in_kwpack", functools.partial(BC.pack_conv_in_kwpack, dtype=H))
    monkeypatch.setattr(SO, "_ulp", _ulp16)
    monkeypatch.setattr(CF, "_ulp", _ulp16)
    monkeypatch.setattr(BC, "_EAGER", _EAGER)      # fp16 eager outputs, apart from the bf16 test's
    return monkeypatch


def test_replay_grid_is_exact_in_fp16():
    g = torch.Generator(device="cuda").manual_seed(0)
    for which in ("x", "w", "b", "os"):
        v = BC._grid((4096,), which, g).double()
        assert torch.equal(v.to(H).double(), v), which


@pytest.mark.parametrize("workload", ["readme", "cfg4"])
def test_f16_bench_step_calls_vs_float64(f16, workload):
    BC.test_bench_step_calls_vs_float64(f16, workload)


@pytest.mark.parametrize("pdl", [False, True])
def test_f16_bench_launch_mode_matches_eager(f16, pdl):
    BC.test_bench_launch_mode_matches_eager(pdl)
