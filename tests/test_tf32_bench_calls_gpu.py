"""Every conv-path kernel call of the benchmark's tokenize + decode on an fp32 model with torch's TF32 switch on, checked one
call at a time against float64 at the benchmark's own shapes: tests/test_bench_calls_gpu.py's three parts (real data call
by call, the exact replay on a dyadic grid with its pipeline defects, the launch mode) on the TF32 kernels.

What changes with TF32 is where the rounding happens.  The tensor core reads each fp32 operand as TF32, its top 19 bits
(DESIGN.md 3.9), so the float64 references run on operands with the low 13 mantissa bits cleared; the products are then
exact and the accumulation allowance is the kernel tests' one.  Outputs are stored in fp32 as computed (half an fp32 ulp;
a SiLU epilogue keeps its exponent's argument rounding, see _forward64_tf32).
The replay grid (x, residual and video in {-8..8} / 2^2, weights in {-8..8} / 2^6, biases in {-64..64} / 2^8, oscale in
{1..8} / 2^3) has at most 4 significant bits, so it is exact in TF32 (test_replay_grid_is_exact_in_tf32) and the replay
still leaves only the epilogue's roundings to allow for.

TF32 has no fused ResidualUnit (DESIGN.md 3.9): every ResidualUnit runs its two convs and squeeze_excite_residual, each
checked on its own.  The pipeline defects (one ring stage missing, the previous tile's accumulators not reset at the
schedule's last tile) must be rejected on the first 64-channel and 512- / 1024-channel 3x3x3 EPI_PLAIN convs and on
conv_out; every slab flavour must run at least one call with more than two tiles per CTA."""
import functools

import pytest
import torch

import synth_data
import tests.test_bench_calls_gpu as BC
import tests.test_conv_forward_gpu as CF
from bench import FRAMES, WORKLOADS
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_NONE, ACT_SILU
from magvit2_pytorch_b200.engine import pack_conv, pack_conv_in_kwpack, pack_ff

pytestmark = pytest.mark.gpu

F32 = torch.float32
_EAGER = {}


def tf32_trunc(t):
    """The TF32 value the tensor core reads of each element of t (fp32-exact values): low 13 mantissa bits cleared."""
    i = t.float().contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32).to(t.dtype)


def _forward64_tf32(x, w, b, os, r, act=ACT_NONE, **kw):
    """CF.forward64 on TF32 operands.  A SiLU epilogue also gets |v| 2^-17: its exponent's argument -z log2(e) rounds
    (|z| 2^-24 relative, |z| < 128 on these calls), which half an ulp of bf16 / fp16 storage absorbs and fp32 does not."""
    ref, acc = CF.forward64(tf32_trunc(x), tf32_trunc(w), b, os, r, act=act, **kw)
    if act == ACT_SILU:
        acc = acc + 2.0 ** -17 * ref.abs()
    return ref, acc


def _geglu64_tf32(x, w1, b1, kern, exact=False):
    return CF.geglu64(tf32_trunc(x), tf32_trunc(w1), b1, kern, exact=exact)


def _workload_tf32(name):
    wl = WORKLOADS[name]
    torch.manual_seed(0)
    model = VideoTokenizer(**wl["kw"])
    synth_data.fill_state_dict_(model, 0)
    model = model.cuda().float().eval()
    clips = wl["clips"] if name == "readme" else 1
    return model, clips, wl["size"]


class _Recorder32(BC._Recorder):
    def residual_unit(self, x, p, ss=None):
        """TF32 ResidualUnits are never fused: their convs and squeeze_excite_residual are checked one by one."""
        assert ss is None
        fused0 = self.eng.fused_ru_calls
        out = self.orig["residual_unit"](x, p)
        assert self.eng.fused_ru_calls == fused0, "a TF32 ResidualUnit ran fused"
        return out


@pytest.fixture
def tf32(monkeypatch):
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    monkeypatch.setattr(BC, "BF", F32)
    monkeypatch.setattr(BC, "_workload", _workload_tf32)
    monkeypatch.setattr(BC, "forward64", _forward64_tf32)
    monkeypatch.setattr(BC, "geglu64", _geglu64_tf32)
    # the replay packs its own grid weights: the wgmma (TF32) layouts of an fp32 model
    monkeypatch.setattr(BC, "pack_conv", functools.partial(pack_conv, tc=True))
    monkeypatch.setattr(BC, "pack_ff", functools.partial(pack_ff, tc=True))
    monkeypatch.setattr(BC, "pack_conv_in_kwpack", functools.partial(pack_conv_in_kwpack, dtype=F32))
    monkeypatch.setattr(BC, "_EAGER", _EAGER)      # TF32 eager outputs, apart from the bf16 test's
    try:
        yield monkeypatch
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev


def test_replay_grid_is_exact_in_tf32():
    g = torch.Generator(device="cuda").manual_seed(0)
    for which in ("x", "w", "b", "os"):
        v = BC._grid((4096,), which, g)
        assert torch.equal(tf32_trunc(v), v), which


def _expected_calls(m):
    """BC._expected_calls with every ResidualUnit unfused."""
    n = BC._expected_calls(m)
    fused = sum(st.count for st in list(m.stages) * 2 if st.kind == "residual" and st.dim in (64, 128))
    n["ru"] -= fused
    n["conv"] += 2 * fused
    n["se"] += fused
    return n


def _defect_targets(calls):
    want = {}
    for c in calls:
        if c.get("flavour") == "plain" and c["pk"].k == (3, 3, 3) and c["pk"].Co in (64, 512, 1024):
            want.setdefault(f"plain C{min(c['pk'].Co, 512)}", id(c))
        elif c.get("flavour") == "ragged_cf":
            want.setdefault("conv_out", id(c))
    return want


@pytest.mark.parametrize("workload", ["readme", "cfg4"])
def test_tf32_bench_step_calls_vs_float64(tf32, workload):
    model, clips, size = _workload_tf32(workload)
    eng = model.engine
    video = synth_data.synth_video(clips, 3, FRAMES, size, seed=1000).cuda()
    rec = _Recorder32(tf32, model)
    with torch.no_grad():
        codes = model.tokenize(video)
        recon = model.decode_from_code_indices(codes)
    torch.cuda.synchronize()
    assert eng.tf32 is False               # reset after the calls
    _EAGER[workload] = (codes.clone(), recon.clone())
    calls = rec.calls
    got = {op: sum(c["op"] == op for c in calls) for op in ("conv", "ru", "se", "rmsnorm", "quantize", "codes")}
    want = _expected_calls(model)
    print(f"\n{workload} TF32: calls checked per kind {got}")
    assert got == want, f"calls per kind {got}, the stages imply {want}"
    assert eng.simt_conv_calls == 0 and not any(c["kind"] == "simt" for c in calls if c["op"] == "conv")
    summ = BC._summary(calls)
    for fl, (n, tot, per) in sorted(summ.items()):
        print(f"  {fl:12s} {n:3d} calls, largest {tot:6d} tiles = {per:3d} tiles per CTA on {rec.n_sm} SMs")
    if workload == "readme":
        assert set(summ) == set(BC.FLAVOURS) - {"ru_c64", "ru_c128"}, sorted(summ)
        few = {fl: per for fl, (n, tot, per) in summ.items() if not any(
            c.get("flavour") == fl and c["plan"]["total"] > 2 * c["plan"]["grid"] for c in calls if "plan" in c)}
        assert not few, f"flavours never run with more than 2 tiles per CTA: {few}"
    targets = _defect_targets(calls)
    ids = set(targets.values())
    gen = torch.Generator(device="cuda").manual_seed(7)
    seen, rejected = set(), {}
    eng.tf32 = True                        # the replays call Engine.conv directly, as a TF32 public call does
    try:
        for c in calls:
            if c["op"] != "conv":
                continue
            key = BC._replay_key(c)
            if key in seen and id(c) not in ids:
                continue
            seen.add(key)
            rec.replay(c, gen, defects=id(c) in ids)
            if id(c) in ids:
                rejected[next(k for k, v in targets.items() if v == id(c))] = c.get("rejected", [])
    finally:
        eng.tf32 = False
    rec._done(0, "allocations outside the checked calls")
    print(f"  {len(seen)} distinct wgmma calls replayed exactly; perturbed references rejected: {rejected}")
    names = {"one ring stage missing", "previous tile's accumulators not reset"}
    assert set(rejected) == {"plain C64", "plain C512", "conv_out"}, rejected
    assert all(set(v) == names for v in rejected.values()), rejected


@pytest.mark.parametrize("pdl", [False, True], ids=["pdl_off", "pdl_on"])
def test_tf32_bench_launch_mode_matches_eager(tf32, pdl):
    BC.test_bench_launch_mode_matches_eager(pdl)
