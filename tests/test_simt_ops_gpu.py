"""The CUDA-core ops of csrc/simt_ops.cu, one C ABI call at a time, against plain float64 torch references (the
oracle/restated.py building blocks where one exists), at the shapes where their dispatch branches: the SqueezeExcite pool
instances and chunk lengths, the vectorised RMSNorm instances and their fallback, the grid-stride loops above their grid
cap, the quantisers' codebook layouts, the LFQ entropy terms, MSE, the gateloop scan, layout / padding and the conditioning
helpers, on both activation dtypes.

Error bounds.  Every input is bf16-representable, so kernel and reference see the same operands.  An output rounded once
to its storage dtype may differ from the float64 value by half an ulp of that dtype (per element, from torch.frexp) plus
an fp32 allowance `acc` for the kernel's arithmetic before that rounding, derived from the kernel's summation depth.  Pure
copies and index outputs must match exactly.  Each op family also checks that its bound rejects a slightly wrong
reference (a dropped row, a mis-split channel range, reversed index digits, a missing token), so a kernel with such a
defect would fail."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R

pytestmark = pytest.mark.gpu

F32, BF16, U8 = 0, 1, 2
DT = {F32: torch.float32, BF16: torch.bfloat16, U8: torch.uint8}
U = 2.0 ** -24                      # fp32 unit roundoff
E_ARG = -1
GRID_CAP = 132 * 32 * 256           # elements one pass of a grid-stride kernel covers (132 SMs x 32 blocks x 256 threads)


def _lib():
    from magvit2_pytorch_b200 import _lib as L
    return L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    from magvit2_pytorch_b200._lib import check
    check(rc, what)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(t):
    """t rounded to bf16, as float64."""
    return t.to(torch.bfloat16).double()


def _randn(shape, g, scale=1.0):
    return _bf(torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) * scale)


def _dev(t64, code):
    return t64.to(DT[code]).contiguous()


def _f32(t):
    return t.float().contiguous()


def _ulp(v, dtype):
    """ulp of |v| in `dtype`, elementwise (float64), 0 where v == 0."""
    p = 8 if dtype == torch.bfloat16 else 24
    _, e = torch.frexp(v.abs())
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - p))


def _excess(out, ref, dtype, acc=0.0):
    """max over elements of |out - ref| - (half an ulp of dtype at |ref| + acc, plus acc); <= 0 means within bound."""
    ref = ref.double()
    acc = torch.as_tensor(acc, dtype=torch.float64, device=ref.device).expand_as(ref)
    bound = 0.5 * _ulp(ref.abs() + acc, dtype) + acc
    return ((out.double().to(ref.device) - ref).abs() - bound).max().item()


def _check(out, ref, dtype, acc=0.0, what=""):
    worst = _excess(out, ref, dtype, acc)
    assert worst <= 0, f"{what}: exceeds its bound by {worst:.3g}"


def _rejects(out, wrong, dtype, acc=0.0, what=""):
    assert _excess(out, wrong, dtype, acc) > 0, f"{what}: the bound does not reject the perturbed reference"


# ------------------------------------------------------------------------------------------------------------------
# SqueezeExcite: mv2_se_pool + mv2_se_gate, mv2_gate_residual, mv2_se_gate_records
# ------------------------------------------------------------------------------------------------------------------
GATE_TOL = 1e-4     # fp32 gates after logit dot, MUFU exp, chunk merge, two small dense layers and a sigmoid


def _se_rows(code, P, C_):
    """Rows per se_pool block (se_rows_per_block): 128 on the generic kernels, P-dependent on the single-pass bf16 one."""
    online = any(C_ % v == 0 and (C_ // v) <= 32 and (C_ // v) & (C_ // v - 1) == 0 for v in (8, 16, 32))
    if code != BF16 or not online:
        return 128
    return 64 if P <= 256 else 128 if P <= 1024 else 512 if P <= 4096 else 2048


def _se_params(C_, Hd, g):
    return dict(wk=_randn(C_, g, C_ ** -0.5), bk=float(_randn(1, g, 0.1)), w1=_randn((Hd, C_), g, 2 * C_ ** -0.5),
                b1=_randn(Hd, g, 0.1), w2=_randn((C_, Hd), g, 2 * Hd ** -0.5), b2=_randn(C_, g, 0.1))


def _se_input(F_, P, C_, rows, prm, g):
    """(F, P, C) activations whose logits are O(0.5) except at the first and last row of every chunk (and of the final
    partial chunk), where they are ~10-12: those rows carry almost all of the softmax mass, so a chunk boundary handled
    wrongly moves the pooled vector, and the gates, by O(0.1)."""
    y = _randn((F_, P, C_), g, 0.5)
    planted = sorted({p for k in range(0, P, rows) for p in (k, min(k + rows, P) - 1)})
    wk = prm["wk"]
    r = torch.randn((F_, len(planted), C_), generator=g, device="cuda", dtype=torch.float64) * 1.5
    target = 10 + 2 * torch.rand((F_, len(planted), 1), generator=g, device="cuda", dtype=torch.float64)
    r = r + (target - r @ wk[:, None] - prm["bk"]) * wk / (wk @ wk)
    y[:, planted] = _bf(r)
    return y, planted


def _se_gates64(y, prm, drop=None):
    """fp64 SqueezeExcite gates of (F, P, C) activations (M:221-240, as R.squeeze_excite), optionally without row `drop`."""
    logit = y @ prm["wk"] + prm["bk"]
    if drop is not None:
        logit[:, drop] = -math.inf
    pooled = torch.einsum("fp,fpc->fc", logit.softmax(dim=-1), y)
    hid = F.leaky_relu(pooled @ prm["w1"].T + prm["b1"], 0.1)
    return torch.sigmoid(hid @ prm["w2"].T + prm["b2"])


def _se_run(y, code, prm, Hd):
    lib = _lib()
    F_, P, C_ = y.shape
    ws = torch.zeros(lib.mv2_se_workspace_bytes(F_, P, C_) // 4, device="cuda", dtype=torch.float32)
    gates = torch.empty((F_, C_), device="cuda", dtype=torch.float32)
    w = {k: _f32(v) for k, v in prm.items() if k != "bk"}
    _ok(lib.mv2_se_pool(y.data_ptr(), code, F_, P, C_, w["wk"].data_ptr(), prm["bk"], ws.data_ptr(), _st()), "mv2_se_pool")
    _ok(lib.mv2_se_gate(ws.data_ptr(), code, F_, P, C_, Hd, w["w1"].data_ptr(), w["b1"].data_ptr(), w["w2"].data_ptr(),
                        w["b2"].data_ptr(), gates.data_ptr(), _st()), "mv2_se_gate")
    nrec = -(-P // _se_rows(code, P, C_))
    return ws[:F_ * nrec * (C_ + 2)].reshape(F_, nrec * (C_ + 2)).clone(), gates


SE_CASES = [
    # every single-pass bf16 instance se_pool_online_kernel<VEC, G> with P > 4096 (2048-row chunks)
    (BF16, 2, 5000, 8, 16), (BF16, 2, 6000, 16, 16), (BF16, 2, 4500, 32, 16), (BF16, 2, 16384, 64, 40),
    (BF16, 2, 16384, 128, 64), (BF16, 2, 16384, 256, 128), (BF16, 2, 5000, 512, 256), (BF16, 2, 4608, 1024, 512),
    # each chunk length (64 / 128 / 512 / 2048 rows) at its edges
    *[(BF16, 3, P, 64, 20) for P in (1, 64, 65, 256, 257, 1024, 1025, 4096, 4097)],
    # the generic bf16 kernel (C not served by a single-pass instance) and the fp32 kernel (128-row chunks)
    (BF16, 2, 300, 24, 16), (BF16, 2, 129, 96, 45), (BF16, 2, 200, 768, 384),
    (F32, 2, 1, 64, 32), (F32, 2, 129, 24, 17), (F32, 2, 1000, 64, 40), (F32, 2, 130, 768, 384),
]


@pytest.mark.parametrize("code,F_,P,C_,Hd", SE_CASES,
                         ids=[f"{'bf16' if c[0] else 'f32'}-F{c[1]}-P{c[2]}-C{c[3]}-Hd{c[4]}" for c in SE_CASES])
def test_squeeze_excite(code, F_, P, C_, Hd):
    g = _gen(P * 7 + C_ * 13 + Hd + code)
    rows = _se_rows(code, P, C_)
    prm = _se_params(C_, Hd, g)
    y64, planted = _se_input(F_, P, C_, rows, prm, g)
    y = _dev(y64, code)
    recs, gates = _se_run(y, code, prm, Hd)
    ref = _se_gates64(y64, prm)
    err = (gates.double() - ref).abs().max().item()
    assert err <= GATE_TOL, f"gates vs fp64: {err:.3g}"
    if P >= 2:      # the last row of the first chunk dropped: the bound must reject it
        wrong = _se_gates64(y64, prm, drop=min(rows, P) - 1)
        assert (gates.double() - wrong).abs().max().item() > GATE_TOL
    # a second call returns identical records and gates (bulk-copy ring refills ordered after the reads they overwrite)
    recs2, gates2 = _se_run(y, code, prm, Hd)
    assert torch.equal(recs, recs2) and torch.equal(gates, gates2)
    # a frame's records and gates do not depend on the other frames of the batch
    for f in range(F_):
        rf, gf = _se_run(y[f:f + 1].contiguous(), code, prm, Hd)
        assert torch.equal(rf[0], recs[f]) and torch.equal(gf[0], gates[f]), f"frame {f} differs batched vs alone"
    # gate_residual on these gates: one fma rounded to fp32, then (bf16) to bf16
    x64 = _randn((F_, P, C_), g)
    x, out = _dev(x64, code), torch.empty_like(y)
    _ok(_lib().mv2_gate_residual(y.data_ptr(), x.data_ptr(), gates.data_ptr(), out.data_ptr(), code, F_, P, C_, _st()),
        "mv2_gate_residual")
    gr = gates.double()[:, None, :] * y64 + x64
    _check(out, gr, DT[code], U * gr.abs() if code == BF16 else 0.0, "gate_residual")


def test_se_reference_matches_oracle():
    """_se_gates64 restates R.squeeze_excite (which returns gates * x): the two agree on a small clip."""
    g = _gen(5)
    prm = _se_params(24, 16, g)
    y = _randn((3, 20, 24), g)
    sd = {"to_k.weight": prm["wk"].reshape(1, 24, 1, 1), "to_k.bias": torch.tensor([prm["bk"]], dtype=torch.float64),
          "net.0.weight": prm["w1"].reshape(16, 24, 1, 1), "net.0.bias": prm["b1"],
          "net.2.weight": prm["w2"].reshape(24, 16, 1, 1), "net.2.bias": prm["b2"]}
    sd = {k: v.cpu() for k, v in sd.items()}
    x5 = y.cpu().reshape(1, 3, 4, 5, 24).permute(0, 4, 1, 2, 3)          # (b, c, f, h, w): 3 frames of 4 x 5
    want = R.squeeze_excite(x5, sd, "").permute(0, 2, 3, 4, 1).reshape(3, 20, 24)
    got = _se_gates64(y, prm).cpu()[:, None, :] * y.cpu()
    assert (got - want).abs().max().item() < 1e-12


GR_CASES = [(BF16, 2, 16384, 160), (BF16, 2, 32768, 25), (F32, 2, 32768, 24)]   # 5.2 M (bf16x8), 1.6 M, 1.6 M elements


@pytest.mark.parametrize("code,F_,P,C_", GR_CASES, ids=["bf16x8", "bf16_scalar", "f32"])
def test_gate_residual_above_grid_cap(code, F_, P, C_):
    """Both grid-stride loops of gate_residual (scalar: 132*32 blocks of 256; bf16x8: 132*16 blocks of 8 x 256) past
    their first pass."""
    assert F_ * P * C_ > (GRID_CAP * 4 if C_ % 8 == 0 and code == BF16 else GRID_CAP)
    g = _gen(F_ + P + C_)
    y64, x64 = _randn((F_, P, C_), g), _randn((F_, P, C_), g)
    gates = torch.rand((F_, C_), generator=g, device="cuda")
    y, x, out = _dev(y64, code), _dev(x64, code), torch.empty((F_, P, C_), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_gate_residual(y.data_ptr(), x.data_ptr(), gates.data_ptr(), out.data_ptr(), code, F_, P, C_, _st()),
        "mv2_gate_residual")
    ref = gates.double()[:, None, :] * y64 + x64
    acc = U * ref.abs() if code == BF16 else 0.0
    _check(out, ref, DT[code], acc, "gate_residual")
    wrong = ref.clone()
    wrong[-1] = gates.double()[0] * y64[-1] + x64[-1]               # the last frame gated with the first frame's gates
    _rejects(out, wrong, DT[code], acc, "gate_residual")


REC_CASES = [(64, 100, 32), (128, 17, 64), (64, 16, 40), (96, 40, 48), (256, 33, 128)]


@pytest.mark.parametrize("C_,nrec,Hd", REC_CASES, ids=[f"C{c}-nrec{n}-Hd{h}" for c, n, h in REC_CASES])
def test_se_gate_records(C_, nrec, Hd):
    """mv2_se_gate_records on hand-built [F][nrec][C + 2] (max, sum, acc[C]) records: se_hidden_kernel<true> for C <= 128
    a power of two with nrec > 16, <false> otherwise."""
    F_ = 3
    g = _gen(C_ + nrec)
    prm = _se_params(C_, Hd, g)
    rows = nrec * 7
    y, _ = _se_input(F_, rows, C_, 7, prm, g)                      # a dominant row at the first and last row of each record
    logit = y @ prm["wk"] + prm["bk"]
    recs = torch.empty((F_, nrec, C_ + 2), device="cuda", dtype=torch.float64)
    for r in range(nrec):
        lr, yr = logit[:, r * 7:(r + 1) * 7], y[:, r * 7:(r + 1) * 7]
        m = lr.max(dim=1).values
        e = torch.exp(lr - m[:, None])
        recs[:, r, 0], recs[:, r, 1], recs[:, r, 2:] = m, e.sum(dim=1), torch.einsum("fp,fpc->fc", e, yr)
    ws = torch.zeros(F_ * nrec * (C_ + 2) + F_ * (C_ + 16), device="cuda", dtype=torch.float32)
    ws[:F_ * nrec * (C_ + 2)] = recs.float().reshape(-1)
    gates = torch.empty((F_, C_), device="cuda", dtype=torch.float32)
    w = {k: _f32(v) for k, v in prm.items() if k != "bk"}
    _ok(_lib().mv2_se_gate_records(ws.data_ptr(), nrec, F_, C_, Hd, w["w1"].data_ptr(), w["b1"].data_ptr(), w["w2"].data_ptr(),
                                   w["b2"].data_ptr(), gates.data_ptr(), _st()), "mv2_se_gate_records")
    ref = _se_gates64(y, prm)
    assert (gates.double() - ref).abs().max().item() <= GATE_TOL
    wrong = _se_gates64(y[:, :-7], prm)                            # the last record left out
    assert (gates.double() - wrong).abs().max().item() > GATE_TOL


# ------------------------------------------------------------------------------------------------------------------
# RMSNorm
# ------------------------------------------------------------------------------------------------------------------
RN_CASES = [
    # code, B, T, P, C, token_shift: n_tok = B*T*P is never a multiple of 32
    (BF16, 2, 3, 37, 64, 0), (BF16, 2, 3, 37, 64, 1), (BF16, 1, 3, 29, 256, 1),        # rmsnorm_bf16x8_kernel<1, 1>
    (BF16, 1, 3, 29, 384, 0), (BF16, 1, 3, 29, 512, 1),                                  # <2, 1>
    (BF16, 2, 3, 13, 1024, 0), (BF16, 2, 3, 13, 1024, 1), (BF16, 1, 5, 7, 768, 1),      # <4, 4>, partial last warp
    (BF16, 1, 3, 21, 36, 0),                       # generic: C % 8 != 0
    (BF16, 1, 3, 11, 1536, 1),                     # generic: C > 1024
    (BF16, 2, 3, 17, 24, 1), (BF16, 1, 4, 9, 40, 1),   # generic: token shift with (C / 2) % 8 != 0
    (BF16, 1, 3, 19, 37, 1),                       # generic, odd C
    (F32, 2, 3, 37, 64, 0), (F32, 2, 3, 37, 64, 1), (F32, 1, 4, 19, 37, 1), (F32, 1, 3, 11, 1030, 1),
]


def _rms_ref(x, gamma, token_shift, half=None):
    """R.token_shift + R.rmsnorm_last on (B, T, P, C); `half` moves the token-shift split (perturbed reference)."""
    if token_shift:
        if half is None:
            x = R.token_shift(x.permute(0, 3, 1, 2)[..., None])[..., 0].permute(0, 2, 3, 1)
        else:
            s = torch.zeros_like(x[..., half:])
            s[:, 1:] = x[:, :-1, :, half:]
            x = torch.cat((x[..., :half], s), dim=-1)
    return R.rmsnorm_last(x, gamma)


@pytest.mark.parametrize("code,B,T,P,C_,ts", RN_CASES,
                         ids=[f"{'bf16' if c[0] else 'f32'}-{c[1]}x{c[2]}x{c[3]}-C{c[4]}-ts{c[5]}" for c in RN_CASES])
def test_rmsnorm(code, B, T, P, C_, ts):
    g = _gen(B * T * P + C_ + ts)
    x64 = _randn((B, T, P, C_), g)
    x64[:, :, 0] = 0                                # pixel 0 is all zero in every frame: the 1e-12 clamp, output exactly 0
    gamma = _randn(C_, g, 0.5) + 1
    x, g32, out = _dev(x64, code), _f32(gamma), torch.empty((B, T, P, C_), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_rmsnorm(x.data_ptr(), out.data_ptr(), code, g32.data_ptr(), B, T, P, C_, ts, _st()), "mv2_rmsnorm")
    ref = _rms_ref(x64, gamma, ts)
    depth = -(-C_ // 32) + 5                        # per-lane fma chain + warp shuffle tree of the sum of squares
    acc = (depth + 6) * U * ref.abs()
    _check(out, ref, DT[code], acc, "rmsnorm")
    assert (out[:, :, 0] == 0).all()
    if ts and C_ % 2:
        _rejects(out, _rms_ref(x64, gamma, ts, half=C_ // 2), DT[code], acc, "rmsnorm token shift split at floor(C/2)")


# ------------------------------------------------------------------------------------------------------------------
# GEGLU
# ------------------------------------------------------------------------------------------------------------------
GG_CASES = [(BF16, 3, 7), (F32, 5, 1), (BF16, 1000, 1365), (F32, 1000, 1365)]


@pytest.mark.parametrize("code,N,I", GG_CASES, ids=[f"{'bf16' if c[0] else 'f32'}-N{c[1]}-I{c[2]}" for c in GG_CASES])
def test_geglu(code, N, I):
    g = _gen(N + I + code)
    inp = _randn((N, 2 * I), g, 2.0)
    src, out = _dev(inp, code), torch.empty((N, I), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_geglu(src.data_ptr(), out.data_ptr(), code, N, I, _st()), "mv2_geglu")
    x, gt = inp[:, :I], inp[:, I:]
    ref = F.gelu(gt) * x
    # erff is within 2 ulp of erf (absolute <= 2^-23 as |erf| < 1), its argument is rounded once: absolute error of
    # (1 + erf) times |0.5 g x|, plus a few roundings relative to the result
    acc = U * (4 * ref.abs() + (3 + 1.2 * gt.abs()) * (0.5 * gt * x).abs())
    _check(out, ref, DT[code], acc, "geglu")
    _rejects(out, F.gelu(x) * gt, DT[code], acc, "geglu with x and gate swapped")


# ------------------------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------------------------
def _quant_params(C_, D, zero_bias, g):
    return dict(win=_randn((D, C_), g, 2 * C_ ** -0.5),
                bin=torch.zeros(D, device="cuda", dtype=torch.float64) if zero_bias else _randn(D, g, 0.1),
                wout=_randn((C_, D), g, D ** -0.5), bout=_randn(C_, g, 0.1))


def _quant_sd(prm, d):
    return {"quantizers.project_in.weight": prm["win"], "quantizers.project_in.bias": prm["bin"],
            "quantizers.project_out.weight": prm["wout"], "quantizers.project_out.bias": prm["bout"],
            "quantizers.mask": 2 ** torch.arange(d - 1, -1, -1, device="cuda")}


def _proj_err(x, prm):
    """fp32 error bound of the kernel's projection (lane-strided fma chain + warp shuffle tree, then + bias)."""
    C_ = x.shape[1]
    return (-(-C_ // 32) + 6) * U * (x.abs() @ prm["win"].abs().T + prm["bin"].abs())


def lfq_presign64(p64, err, nc, d, spherical):
    """(reference, allowance) of the LFQ kernel's fp32 pre-sign values from the float64 projection p64 (N, nc d) and its
    error bound err: p64 itself, or per codebook L2-normalised when spherical (a zero vector stays zero)."""
    if not spherical:
        return p64, err
    N = p64.shape[0]
    pc = p64.reshape(N, nc, d)
    nrm = pc.norm(dim=-1, keepdim=True)
    pn = torch.where(nrm > 0, pc / nrm.clamp(min=1e-300), torch.zeros_like(pc))
    en = torch.where(nrm > 0, 2 * err.reshape(N, nc, d).max(dim=-1, keepdim=True).values * d ** 0.5 / nrm.clamp(min=1e-300)
                     + (d + 8) * U, torch.zeros_like(nrm))
    return pn.reshape(N, nc * d), en.expand(N, nc, d).reshape(N, nc * d)


LFQ_CASES = [
    # code, d, nc, spherical, clamp, zero bias, C
    (BF16, 16, 1, 0, 10.0, 1, 40), (F32, 16, 1, 1, 10.0, 0, 40),
    (F32, 8, 2, 1, 10.0, 1, 136), (BF16, 8, 2, 0, 0.0, 0, 136),
    (BF16, 4, 4, 1, 0.0, 1, 40), (F32, 4, 4, 0, 10.0, 0, 40),
    (F32, 5, 3, 0, 0.0, 1, 72), (BF16, 5, 3, 1, 10.0, 0, 72),
]


@pytest.mark.parametrize("code,d,nc,sph,clamp,zb,C_", LFQ_CASES,
                         ids=[f"{'bf16' if c[0] else 'f32'}-{c[1]}x{c[2]}-sph{c[3]}-clamp{c[4]:g}-zb{c[5]}" for c in LFQ_CASES])
def test_lfq(code, d, nc, sph, clamp, zb, C_):
    lib = _lib()
    N, D = 1003, d * nc
    g = _gen(d * 100 + nc * 10 + sph + C_)
    prm = _quant_params(C_, D, zb, g)
    x64 = _randn((N, C_), g)
    zero_rows = torch.arange(0, N, 97, device="cuda")
    x64[zero_rows] = 0
    x = _dev(x64, code)
    idx = torch.empty((N, nc), device="cuda", dtype=torch.int64)
    q = torch.empty((N, C_), device="cuda", dtype=DT[code])
    pre = torch.empty((N, D), device="cuda", dtype=torch.float32)
    w = {k: _f32(v) for k, v in prm.items()}
    _ok(lib.mv2_lfq_forward(x.data_ptr(), code, N, C_, d, nc, w["win"].data_ptr(), w["bin"].data_ptr(), w["wout"].data_ptr(),
                            w["bout"].data_ptr(), clamp, sph, idx.data_ptr(), q.data_ptr(), pre.data_ptr(), _st()),
        "mv2_lfq_forward")
    sd = _quant_sd(prm, d)
    x5 = x64.T.reshape(1, C_, N, 1, 1)
    q_ref, idx_ref, _ = R.lfq_quantize(x5, sd, clamp if clamp > 0 else None, nc, bool(sph))
    q_ref, idx_ref = q_ref.reshape(C_, N).T, idx_ref.reshape(N, nc)
    # fp64 pre-sign values (R.lfq_presign returns them rounded to fp32) and the kernel's error bound on them
    lin = x64 @ prm["win"].T + prm["bin"]
    err = _proj_err(x64, prm)
    p64 = torch.tanh(lin / clamp) * clamp if clamp > 0 else lin
    err = err + 4 * U * p64.abs()
    ambiguous = ((p64.abs() < err).reshape(N, nc, d).any(dim=-1))            # sign within fp32 noise of 0
    assert ambiguous.sum().item() <= max(2, N // 100)
    assert torch.equal(idx[~ambiguous], idx_ref[~ambiguous])
    if zb:
        assert (idx[zero_rows] == 0).all()
    # the bound rejects the index bits taken in reversed order
    rev = torch.zeros_like(idx_ref)
    for j in range(d):
        rev |= ((idx_ref >> j) & 1) << (d - 1 - j)
    assert (idx != rev).sum().item() > ambiguous.sum().item()
    # pre-sign values: fp32 projection (+ tanh clamp), per codebook L2-normalised when spherical
    pre_ref, pre_acc = lfq_presign64(p64, err, nc, d, sph)
    _check(pre, pre_ref, torch.float32, pre_acc, "lfq presign" + (" (spherical)" if sph else ""))
    # quantized: bout + Wout (+-1) as a D-term fp32 fma chain, rounded once
    acc = (D + 1) * U * (prm["wout"].abs().sum(dim=1) + prm["bout"].abs())
    ok = ~ambiguous.any(dim=1)
    _check(q[ok], q_ref[ok], DT[code], acc.expand(N, C_)[ok], "lfq quantized")
    # decode of the forward's own indices (int64 and int32) reproduces its quantized output bit for bit
    for is64, ii in ((1, idx), (0, idx.int().contiguous())):
        qd = torch.empty_like(q)
        _ok(lib.mv2_lfq_decode(ii.data_ptr(), is64, N, C_, d, nc, w["wout"].data_ptr(), w["bout"].data_ptr(), qd.data_ptr(),
                               code, _st()), "mv2_lfq_decode")
        assert torch.equal(qd, q)
    # decode of every code (d <= 12; a spread of codes with both extremes above that) in every codebook
    K = 2 ** d
    base = torch.arange(K, device="cuda") if d <= 12 else torch.cat((torch.tensor([0, K - 1], device="cuda"),
                                                                    torch.randint(0, K, (2046,), generator=g, device="cuda")))
    codes = torch.stack([(base + cb * (K // 3)) % K for cb in range(nc)], dim=1).contiguous()
    M = codes.shape[0]
    want = R.lfq_indices_to_codes(codes if nc > 1 else codes[:, 0], sd, torch.float64, nc)
    outs = []
    for is64, ii in ((1, codes), (0, codes.int().contiguous())):
        qd = torch.empty((M, C_), device="cuda", dtype=DT[code])
        _ok(lib.mv2_lfq_decode(ii.data_ptr(), is64, M, C_, d, nc, w["wout"].data_ptr(), w["bout"].data_ptr(), qd.data_ptr(),
                               code, _st()), "mv2_lfq_decode")
        outs.append(qd)
    assert torch.equal(outs[0], outs[1])
    _check(outs[0], want, DT[code], acc.expand(M, C_), "lfq decode")


def fsq64(x64, prm, levels, nc):
    """float64 FSQ of tokens x64 (N, C) with projections prm (oracle.restated.fsq_quantize) and the kernel's allowances:
    dict(q, idx (N, nc), bounded (N, nc d), err: the allowance of the fp32 bounded values, ambiguous (N, nc): a bounded
    value within err of a .5 rounding point (its digit may round either way), reversed: the indices with the mixed-radix
    digits in reverse order (first dimension most significant), acc_q: the allowance of the quantized output per channel
    before its rounding)."""
    N, C_ = x64.shape
    d = len(levels)
    D = d * nc
    sd = {k: v.cpu() for k, v in _quant_sd(prm, d).items()}        # R's FSQ constants are CPU tensors
    q_ref, idx_ref, b_ref = R.fsq_quantize(x64.T.reshape(1, C_, N, 1, 1).cpu(), sd, levels, nc)
    q_ref, idx_ref, b_ref = q_ref.reshape(C_, N).T.cuda(), idx_ref.reshape(N, nc).cuda(), b_ref.reshape(N, D).cuda()
    # bounded = tanh(z + shift) * half_l - offset: the projection error, scaled by half_l, plus a few roundings
    half_l = torch.tensor([(l - 1) * 1.001 / 2 for l in levels] * nc, device="cuda", dtype=torch.float64)
    lin = x64 @ prm["win"].T + prm["bin"]
    err = half_l * (_proj_err(x64, prm) + 8 * U * (1 + lin.abs()))
    frac = b_ref - torch.floor(b_ref)
    ambiguous = ((frac - 0.5).abs() < err).reshape(N, nc, d).any(dim=-1)
    digits = torch.round(b_ref).reshape(N, nc, d) + torch.tensor([l // 2 for l in levels], device="cuda")
    rbasis = [math.prod(levels[j + 1:]) for j in range(d)]
    rev = (digits * torch.tensor(rbasis, device="cuda", dtype=torch.float64)).sum(dim=-1).to(torch.int32)
    acc = (D + 2) * U * (prm["wout"].abs().sum(dim=1) + prm["bout"].abs())
    return dict(q=q_ref, idx=idx_ref, bounded=b_ref, err=err, ambiguous=ambiguous, reversed=rev, acc_q=acc)


FSQ_CASES = [
    (BF16, [2] * 16, 1), (F32, [2] * 16, 1),
    (F32, [3, 2, 4, 5, 2, 3, 2, 2], 2), (BF16, [3, 2, 4, 5, 2, 3, 2, 2], 2),
    (BF16, [8, 5, 5, 5], 4), (F32, [8, 5, 5, 5], 4),
    (F32, [7, 5, 6, 2, 5], 3), (BF16, [7, 5, 6, 2, 5], 3),
]


@pytest.mark.parametrize("code,levels,nc", FSQ_CASES,
                         ids=[f"{'bf16' if c[0] else 'f32'}-{'.'.join(map(str, c[1]))}x{c[2]}" for c in FSQ_CASES])
def test_fsq(code, levels, nc):
    lib = _lib()
    d = len(levels)
    N, D, C_ = 1003, d * nc, 40 if nc != 2 else 136
    g = _gen(sum(levels) * 10 + nc + code)
    prm = _quant_params(C_, D, nc % 2, g)
    prm["win"] = prm["win"] * 1.5
    x64 = _randn((N, C_), g)
    x64[::97] = 0
    lv = (C.c_int32 * d)(*levels)
    idx = torch.empty((N, nc), device="cuda", dtype=torch.int32)
    q = torch.empty((N, C_), device="cuda", dtype=DT[code])
    bnd = torch.empty((N, D), device="cuda", dtype=torch.float32)
    w = {k: _f32(v) for k, v in prm.items()}
    x = _dev(x64, code)
    _ok(lib.mv2_fsq_forward(x.data_ptr(), code, N, C_, d, nc, lv, w["win"].data_ptr(), w["bin"].data_ptr(),
                            w["wout"].data_ptr(), w["bout"].data_ptr(), idx.data_ptr(), q.data_ptr(), bnd.data_ptr(), _st()),
        "mv2_fsq_forward")
    f = fsq64(x64, prm, levels, nc)
    sd = {k: v.cpu() for k, v in _quant_sd(prm, d).items()}        # R's FSQ constants are CPU tensors
    _check(bnd, f["bounded"], torch.float32, f["err"], "fsq bounded")
    ambiguous = f["ambiguous"]
    assert ambiguous.sum().item() <= max(2, N // 100)
    assert torch.equal(idx[~ambiguous], f["idx"][~ambiguous])
    # the bound rejects the mixed-radix digits taken in reversed order (first dimension most significant)
    assert (idx != f["reversed"]).sum().item() > ambiguous.sum().item()
    acc = f["acc_q"]
    ok = ~ambiguous.any(dim=1)
    _check(q[ok], f["q"][ok], DT[code], acc.expand(N, C_)[ok], "fsq quantized")
    for is64, ii in ((0, idx), (1, idx.long().contiguous())):
        qd = torch.empty_like(q)
        _ok(lib.mv2_fsq_decode(ii.data_ptr(), is64, N, C_, d, nc, lv, w["wout"].data_ptr(), w["bout"].data_ptr(), qd.data_ptr(),
                               code, _st()), "mv2_fsq_decode")
        assert torch.equal(qd, q)
    # every code of the codebook, in every codebook
    K = math.prod(levels)
    codes = torch.stack([(torch.arange(K, device="cuda") + cb * (K // 3)) % K for cb in range(nc)], dim=1).int().contiguous()
    want = R.fsq_indices_to_codes((codes if nc > 1 else codes[:, 0]).cpu(), sd, levels, torch.float64, nc).cuda()
    outs = []
    for is64, ii in ((0, codes), (1, codes.long().contiguous())):
        qd = torch.empty((K, C_), device="cuda", dtype=DT[code])
        _ok(lib.mv2_fsq_decode(ii.data_ptr(), is64, K, C_, d, nc, lv, w["wout"].data_ptr(), w["bout"].data_ptr(), qd.data_ptr(),
                               code, _st()), "mv2_fsq_decode")
        outs.append(qd)
    assert torch.equal(outs[0], outs[1])
    _check(outs[0], want, DT[code], acc.expand(K, C_), "fsq decode")


# ------------------------------------------------------------------------------------------------------------------
# LFQ training terms: mv2_lfq_entropy_partials, mv2_lfq_aux_finalize
# ------------------------------------------------------------------------------------------------------------------
def _lfq_entropy64(p, d, inv_t):
    """fp64 A.1 steps 7-8 on pre-sign values p (N, nc, d): (sum of per-token entropies, sum (p - sign p)^2,
    un-normalised avg_prob (nc, K)) -- R.lfq_train_losses computes the same in fp32."""
    K = 2 ** d
    mask = 2 ** torch.arange(d - 1, -1, -1, device=p.device)
    cb = ((torch.arange(K, device=p.device)[:, None] & mask) != 0).double() * 2 - 1
    prob = (2 * inv_t * torch.einsum("tcd,kd->tck", p, cb)).softmax(dim=-1)
    ent = (-prob * torch.log(prob.clamp(min=1e-5))).sum(dim=-1)
    q = torch.where(p > 0, torch.ones_like(p), -torch.ones_like(p))
    return ent.sum(), ((p - q) ** 2).sum(), prob.sum(dim=0)


def _entropy_run(p, d, nc, inv_t):
    N = p.shape[0]
    avg = torch.zeros((nc, 2 ** d), device="cuda", dtype=torch.float32)
    stats = torch.zeros(2, device="cuda", dtype=torch.float32)
    p32 = _f32(p)
    _ok(_lib().mv2_lfq_entropy_partials(p32.data_ptr(), N, d, nc, inv_t, avg.data_ptr(), stats.data_ptr(), _st()),
        "mv2_lfq_entropy_partials")
    return avg, stats


ENT_CASES = [(1, 1, 5, 100.0), (3, 2, 31, 1.0), (8, 4, 45, 100.0), (9, 1, 70, 1.0), (12, 2, 33, 100.0), (12, 1, 3, 1.0)]


@pytest.mark.parametrize("d,nc,N,inv_t", ENT_CASES, ids=[f"d{c[0]}-nc{c[1]}-N{c[2]}-it{c[3]:g}" for c in ENT_CASES])
def test_lfq_entropy_and_finalize(d, nc, N, inv_t):
    g = _gen(d * 1000 + nc * 100 + N)
    # multiples of 2^-8 in [-1, 1]: the kernel's code logits 2 inv_t <p, code> are then exact in fp32
    p = torch.randint(-256, 257, (N, nc, d), generator=g, device="cuda").double() / 256
    p[-1] = 0                                     # the last token is uniform over the codes: the largest entropy
    avg, stats = _entropy_run(p, d, nc, inv_t)
    ent, com, prob = _lfq_entropy64(p, d, inv_t)
    K, nblk = 2 ** d, -(-N // 32)
    # fp32 roundings: exp / reciprocal / log per code, the K-term sums, 32 tokens per block, one atomic per warp / block
    rel = (K // 256 + 80 + 8 * nblk) * U
    tol0 = rel * (ent.item() + N * nc)
    assert abs(stats[0].item() - ent.item()) <= tol0, (stats[0].item(), ent.item())
    assert abs(stats[1].item() - com.item()) <= (d + 40 + nblk) * U * com.item()
    assert ((avg.double() - prob).abs() <= rel * prob + 1e-36 * N).all()
    # the bound rejects the entropy of the last token left out
    ent_wrong, _, _ = _lfq_entropy64(p[:-1], d, inv_t)
    assert abs(stats[0].item() - ent_wrong.item()) > tol0
    # finalize on two halves of the tokens, avg_prob summed as the cross-rank all-reduce would: world size 2
    if N >= 2:
        h = N // 2
        a0, s0 = _entropy_run(p[:h], d, nc, inv_t)
        a1, _ = _entropy_run(p[h:2 * h], d, nc, inv_t)
        out4, asum = torch.empty(4, device="cuda", dtype=torch.float32), a0 + a1
        _ok(_lib().mv2_lfq_aux_finalize(asum.data_ptr(), s0.data_ptr(), d, nc, h, 2 * h, 2.5, 0.1, 1.0, out4.data_ptr(),
                                        _st()), "mv2_lfq_aux_finalize")
        p0, p1 = p[:h].float().cpu().reshape(1, h, nc * d), p[h:2 * h].float().cpu().reshape(1, h, nc * d)
        avg1 = R.lfq_train_losses(p1, d, inv_temperature=inv_t, nc=nc)[4]
        want = R.lfq_train_losses(p0, d, world_reduce=lambda a: (a + avg1) / 2, inv_temperature=inv_t, nc=nc)[:4]
        got = out4.cpu().tolist()
        ps, be, cm, aux = [w.item() for w in want]
        scale = [abs(ps), abs(be), abs(cm), 0.1 * abs(ps) + 0.25 * abs(be) + abs(cm)]
        for k in range(4):
            assert abs(got[k] - [ps, be, cm, aux][k]) <= 1e-4 * scale[k] + 1e-6, (k, got, [ps, be, cm, aux])


# ------------------------------------------------------------------------------------------------------------------
# MSE
# ------------------------------------------------------------------------------------------------------------------
MSE_PAIRS = [(F32, F32), (F32, BF16), (BF16, F32), (BF16, BF16), (U8, F32), (U8, BF16)]
MSE_N = [1, 255, 256, 257, 592 * 256 * 4 + 1, 20_000_003]


@pytest.mark.parametrize("n", MSE_N)
@pytest.mark.parametrize("ad,bd", MSE_PAIRS, ids=["f32-f32", "f32-bf16", "bf16-f32", "bf16-bf16", "u8-f32", "u8-bf16"])
def test_mse(ad, bd, n):
    lib = _lib()
    g = _gen(n + 10 * ad + bd)
    if ad == U8:
        a = torch.randint(0, 256, (n,), generator=g, device="cuda", dtype=torch.uint8)
        a64 = a.double() / 255
        b64 = _bf(torch.rand(n, generator=g, device="cuda", dtype=torch.float64))
    else:
        a64 = _randn(n, g)
        a = _dev(a64, ad)
        b64 = _randn(n, g)
    b64[-1] = _bf(a64[-1] + 256)               # a planted large last term: dropping it is visible at every n
    b = _dev(b64, bd)
    ws = torch.empty(lib.mv2_mse_workspace_bytes(), device="cuda", dtype=torch.uint8)
    outs = []
    for _ in range(2):
        out = torch.empty(1, device="cuda", dtype=torch.float32)
        _ok(lib.mv2_mse(a.data_ptr(), ad, b.data_ptr(), bd, n, ws.data_ptr(), out.data_ptr(), _st()), "mv2_mse")
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "mv2_mse is not repeatable"
    dl = a64 - b64
    ref = (dl * dl).mean()
    steps = -(-n // (min(592, -(-n // 256)) * 256))           # fp32 fma steps per thread
    # fp32 difference and fma chain relative to the sum, the u8 -> fp32 division (one rounding of a), the fp32 output
    tol = (steps + 6) * U * ref + 3 * U * (a64.abs() * dl.abs()).mean()
    assert abs(outs[0].double().item() - ref.item()) <= tol.item(), (outs[0].item(), ref.item())
    if n >= 2:
        wrong = (dl[:-1] * dl[:-1]).mean()
        assert abs(outs[0].double().item() - wrong.item()) > tol.item()


# ------------------------------------------------------------------------------------------------------------------
# gateloop scan
# ------------------------------------------------------------------------------------------------------------------
def gateloop64(qkva, res):
    """float64 gateloop recurrence of mv2_gateloop_scan on (B, T, P, 3C) qkva and (B, T, P, C) res: s_t = sigmoid(a_t) s_{t-1}
    + kv_t, out_t = q_t s_t + res_t.  Returns (reference, allowance, wrong): the allowance carries a running bound on the
    fp32 state error; `wrong` takes each output from the state before that step's update."""
    C_, T = res.shape[-1], res.shape[1]
    q, kv, sg = qkva[..., :C_], qkva[..., C_:2 * C_], torch.sigmoid(qkva[..., 2 * C_:])
    s = torch.zeros_like(q[:, 0])
    mag, err = torch.zeros_like(s), torch.zeros_like(s)
    ref, acc, wrong = torch.empty_like(res), torch.empty_like(res), torch.empty_like(res)
    for t in range(T):
        wrong[:, t] = q[:, t] * s + res[:, t]
        s = sg[:, t] * s + kv[:, t]
        mag = sg[:, t] * mag + kv[:, t].abs()
        err = sg[:, t] * err + 6 * U * mag                     # sigmoid (expf, add, divide) and the fma, per step
        ref[:, t] = q[:, t] * s + res[:, t]
        acc[:, t] = q[:, t].abs() * err + U * ((q[:, t] * s).abs() + res[:, t].abs())
    return ref, acc, wrong


GL_CASES = [(F32, 2, 1, 37, 7), (BF16, 1, 1, 45, 13), (F32, 2, 17, 100, 24), (BF16, 1, 17, 45, 13), (BF16, 2, 5, 300, 40)]


@pytest.mark.parametrize("code,B,T,P,C_", GL_CASES, ids=[f"{'bf16' if c[0] else 'f32'}-{c[1]}x{c[2]}x{c[3]}-C{c[4]}" for c in GL_CASES])
def test_gateloop_scan(code, B, T, P, C_):
    assert (B * P * C_) % 256 != 0
    g = _gen(B * T * P * C_)
    qkva = _randn((B, T, P, 3 * C_), g)
    a = qkva[..., 2 * C_:]
    sat = torch.rand(a.shape, generator=g, device="cuda") < 0.3
    sign = torch.where(torch.rand(a.shape, generator=g, device="cuda") < 0.5, 1.0, -1.0).double()
    a[sat] = 30 * sign[sat]                                                                    # saturated gates
    res = _randn((B, T, P, C_), g)
    qd, rd, out = _dev(qkva, code), _dev(res, code), torch.empty((B, T, P, C_), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_gateloop_scan(qd.data_ptr(), rd.data_ptr(), out.data_ptr(), code, B, T, P, C_, _st()), "mv2_gateloop_scan")
    ref, acc, wrong = gateloop64(qkva, res)
    _check(out, ref, DT[code], acc, "gateloop")
    if T > 1:
        _rejects(out, wrong, DT[code], acc, "gateloop with the output taken from the previous state")


# ------------------------------------------------------------------------------------------------------------------
# layout and padding: exact
# ------------------------------------------------------------------------------------------------------------------
LAYOUT_PAIRS = [(s, d_) for s in (F32, BF16, U8) for d_ in (F32, BF16)]


def _src(shape, code, g):
    if code == U8:
        u = torch.randint(0, 256, shape, generator=g, device="cuda", dtype=torch.uint8)
        # x / 255 correctly rounded to fp32 (torch's CUDA division by a scalar multiplies by its reciprocal instead)
        return u, (u.double() / 255).float()
    v = _randn(shape, g)
    return _dev(v, code), v.float()


@pytest.mark.parametrize("sd_,dd", LAYOUT_PAIRS, ids=[f"{'f32 bf16 u8'.split()[s]}-{'f32 bf16'.split()[d_]}" for s, d_ in LAYOUT_PAIRS])
def test_to_channels_last_and_first(sd_, dd):
    lib = _lib()
    B, C_, T, H, W, tp = 2, 40, 5, 7, 33, 2
    g = _gen(sd_ * 3 + dd)
    src, val = _src((B, C_, T, H, W), sd_, g)
    dst = torch.full((B, T + tp, H, W, C_), 7.0, device="cuda", dtype=DT[dd])
    _ok(lib.mv2_to_channels_last(src.data_ptr(), sd_, dst.data_ptr(), dd, B, C_, T, H, W, tp, _st()), "mv2_to_channels_last")
    want = F.pad(val.permute(0, 2, 3, 4, 1), (0, 0, 0, 0, 0, 0, tp, 0)).to(DT[dd])
    assert torch.equal(dst, want)
    # channels-last -> channels-first with the first frames cropped
    s2, v2 = _src((B, T, H, W, C_), sd_, g)
    crop = 3
    out = torch.empty((B, C_, T - crop, H, W), device="cuda", dtype=DT[dd])
    _ok(lib.mv2_to_channels_first(s2.data_ptr(), sd_, out.data_ptr(), dd, B, C_, T, H, W, crop, _st()), "mv2_to_channels_first")
    assert torch.equal(out, v2[:, crop:].permute(0, 4, 1, 2, 3).to(DT[dd]))


def test_copy_frames_zero_front():
    lib = _lib()
    B, sT, dT, fb = 2, 6, 9, 5 * 3 * 8
    src = torch.randn((B, sT, 5, 3, 8), device="cuda").to(torch.bfloat16)
    dst = torch.full((B, dT, 5, 3, 8), 3.0, device="cuda", dtype=torch.bfloat16)
    _ok(lib.mv2_copy_frames(src.data_ptr(), dst.data_ptr(), B, sT, dT, 1, 4, 4, fb * 2, 1, _st()), "mv2_copy_frames")
    want = torch.full_like(dst, 3.0)
    want[:, :4] = 0
    want[:, 4:8] = src[:, 1:5]
    assert torch.equal(dst, want)


@pytest.mark.parametrize("W", [31, 130])
@pytest.mark.parametrize("sd_", [F32, BF16, U8], ids=["f32", "bf16", "u8"])
def test_ingest_kwpack(sd_, W):
    B, C_, T, H, tp, kw, pw, cpack = 2, 3, 4, 5, 2, 7, 3, 32
    g = _gen(W + sd_)
    src, val = _src((B, C_, T, H, W), sd_, g)
    dst = torch.full((B, T + tp, H, W, cpack), 5.0, device="cuda", dtype=torch.bfloat16)
    _ok(_lib().mv2_ingest_kwpack(src.data_ptr(), sd_, dst.data_ptr(), B, C_, T, H, W, tp, kw, pw, cpack, _st()),
        "mv2_ingest_kwpack")
    xp = F.pad(val.permute(0, 2, 3, 4, 1), (0, 0, pw, kw - 1 - pw, 0, 0, tp, 0))      # (B, T+tp, H, W+kw-1, C)
    want = torch.zeros((B, T + tp, H, W, cpack), device="cuda")
    for dw in range(kw):
        want[..., dw * C_:(dw + 1) * C_] = xp[:, :, :, dw:dw + W]
    assert torch.equal(dst, want.to(torch.bfloat16))


PAD_CASES = [
    # mode, (B, T, H, W, C), (pt, ph, pw)
    (1, (2, 3, 4, 5, 6), (2, 3, 4)),        # reflect at its largest legal pad: size - 1
    (3, (2, 3, 4, 5, 6), (3, 4, 5)),        # circular at its largest legal pad: size
    (2, (2, 1, 4, 5, 6), (2, 2, 3)),        # replicate with T = 1
    (2, (1, 4, 64, 64, 64), (2, 1, 1)),     # 1.2 M elements: past the first grid-stride pass
]


@pytest.mark.parametrize("code", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("mode,shape,pad", PAD_CASES, ids=["reflect", "circular", "replicate_T1", "replicate_big"])
def test_pad_cl(mode, shape, pad, code):
    B, T, H, W, C_ = shape
    pt, ph, pw = pad
    g = _gen(mode + T + code)
    x = _dev(_randn(shape, g), code)
    out = torch.empty((B, T + pt, H + 2 * ph, W + 2 * pw, C_), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_pad_cl(x.data_ptr(), out.data_ptr(), code, B, T, H, W, C_, pt, ph, pw, mode, _st()), "mv2_pad_cl")
    name = {1: "reflect", 2: "replicate", 3: "circular"}[mode]
    want = F.pad(x.float().permute(0, 4, 1, 2, 3), (pw, pw, ph, ph, pt, 0), mode=name).permute(0, 2, 3, 4, 1)
    assert torch.equal(out, want.to(DT[code]))


# ------------------------------------------------------------------------------------------------------------------
# conditioning helpers
# ------------------------------------------------------------------------------------------------------------------
ACTS = {0: lambda v: v, 1: F.elu, 2: F.silu, 3: lambda v: F.leaky_relu(v, 0.1)}


def dense_small64(x, w, b, act):
    """(reference, allowance, pre-activation) of mv2_dense_small: act(x w^T + b) in float64 (b may be None); the
    allowance covers the lane fma chain, shuffle tree and bias, then the activation (Lipschitz <= 1.1, a few ulp of libm)."""
    K = x.shape[1]
    lin = x @ w.T + (0 if b is None else b)
    ref = ACTS[act](lin)
    acc = 1.1 * (-(-K // 32) + 7) * U * ((x.abs() @ w.abs().T) + (0 if b is None else b.abs())) + 4 * U * ref.abs()
    return ref, acc, lin


def mod_prepare64(cond, S, eps):
    """(scale_in, inv_norm, inv_norm allowance, the wrong inv_norm with eps on the norm) of mv2_mod_prepare in float64 from
    its fp32 inputs: scale_in = cond + 1 (one fp32 rounding), inv_norm = rsqrt(max((cond + 1)^2 . S, eps)); the allowance
    covers (cond + 1)^2, the fma chain relative to a positive sum, and rsqrtf."""
    ssum = ((cond + 1) ** 2) @ S.T
    ref = torch.rsqrt(ssum.clamp(min=eps))
    acc = (-(-cond.shape[1] // 32) + 12) * U * ref
    return cond + 1, ref, acc, 1 / ssum.sqrt().clamp(min=eps)


def scale_channels64(x, sc, dtype):
    """(reference, allowance) of mv2_scale_channels: x (B, P, C) times the per-clip channel scale sc (B, C), one fp32
    product rounded to dtype (the fp32 output rounds exactly once, the bf16 one after the fp32 product)."""
    ref = x * sc[:, None, :]
    return ref, (U * ref.abs() if dtype == torch.bfloat16 else 0.0)


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("act", [0, 1, 2, 3], ids=["none", "elu", "silu", "leaky"])
def test_dense_small(act, bias):
    B, K, N = 3, 50, 77
    g = _gen(act * 2 + bias)
    x, w = _randn((B, K), g), _randn((N, K), g, K ** -0.5)
    b = _randn(N, g, 0.5) if bias else None
    y = torch.empty((B, N), device="cuda", dtype=torch.float32)
    x32, w32, b32 = _f32(x), _f32(w), (_f32(b) if bias else None)
    _ok(_lib().mv2_dense_small(x32.data_ptr(), w32.data_ptr(), b32.data_ptr() if bias else None, y.data_ptr(), B, K, N, act,
                               _st()), "mv2_dense_small")
    ref, acc, lin = dense_small64(x, w, b, act)
    _check(y, ref, torch.float32, acc, "dense_small")
    if act == 3:
        _rejects(y, F.leaky_relu(lin, 0.01), torch.float32, acc, "dense_small with torch's default leaky slope")


def test_mod_prepare():
    B, Ci, Co, eps = 3, 70, 45, 1e-8
    g = _gen(11)
    cond = _randn((B, Ci), g, 0.5)
    S = _randn((Co, Ci), g).abs() * 0.01
    S[5] = 0                                         # output channel 5: sum 0, floored at eps
    si = torch.empty((B, Ci), device="cuda", dtype=torch.float32)
    inv = torch.empty((B, Co), device="cuda", dtype=torch.float32)
    c32, s32 = _f32(cond), _f32(S)
    _ok(_lib().mv2_mod_prepare(c32.data_ptr(), s32.data_ptr(), eps, si.data_ptr(), inv.data_ptr(), B, Ci, Co, _st()),
        "mv2_mod_prepare")
    si_ref, ref, acc, wrong = mod_prepare64(cond, S, eps)
    _check(si, si_ref, torch.float32, 0.0, "mod_prepare scale_in")
    _check(inv, ref, torch.float32, acc, "mod_prepare inv_norm")
    assert abs(inv[0, 5].item() - eps ** -0.5) <= 8 * U * eps ** -0.5
    _rejects(inv, wrong, torch.float32, acc, "mod_prepare with eps on the norm")


@pytest.mark.parametrize("code", [F32, BF16], ids=["f32", "bf16"])
def test_scale_channels_above_grid_cap(code):
    B, Pn, C_ = 2, 40000, 24
    assert B * Pn * C_ > GRID_CAP
    g = _gen(code + 3)
    x = _randn((B, Pn, C_), g)
    sc = _randn((B, C_), g)
    xd, s32, out = _dev(x, code), _f32(sc), torch.empty((B, Pn, C_), device="cuda", dtype=DT[code])
    _ok(_lib().mv2_scale_channels(xd.data_ptr(), s32.data_ptr(), out.data_ptr(), code, B, Pn, C_, _st()), "mv2_scale_channels")
    ref, acc = scale_channels64(x, sc, DT[code])
    _check(out, ref, DT[code], acc, "scale_channels")
    _rejects(out, x * sc[:1, None, :], DT[code], acc, "scale_channels with clip 0's scale everywhere")


# ------------------------------------------------------------------------------------------------------------------
# programmatic dependent launch, host-side argument checks
# ------------------------------------------------------------------------------------------------------------------
def test_pdl_chain_bitwise():
    """rmsnorm -> se_pool -> se_gate -> gate_residual -> mse with programmatic dependent launch on gives bit-identical
    results to the plain stream order."""
    lib = _lib()
    T, P, C_, Hd = 3, 4608, 64, 32
    g = _gen(17)
    x = _randn((1, T, P, C_), g).to(torch.bfloat16)
    gamma = _f32(_randn(C_, g, 0.5) + 1)
    prm = {k: (_f32(v) if k != "bk" else v) for k, v in _se_params(C_, Hd, g).items()}

    def run():
        st = _st()
        y = torch.empty_like(x)
        ws = torch.zeros(lib.mv2_se_workspace_bytes(T, P, C_) // 4, device="cuda", dtype=torch.float32)
        gates = torch.empty((T, C_), device="cuda", dtype=torch.float32)
        out = torch.empty_like(x)
        mws = torch.empty(lib.mv2_mse_workspace_bytes(), device="cuda", dtype=torch.uint8)
        loss = torch.empty(1, device="cuda", dtype=torch.float32)
        torch.cuda.synchronize()
        _ok(lib.mv2_rmsnorm(x.data_ptr(), y.data_ptr(), BF16, gamma.data_ptr(), 1, T, P, C_, 1, st), "mv2_rmsnorm")
        _ok(lib.mv2_se_pool(y.data_ptr(), BF16, T, P, C_, prm["wk"].data_ptr(), prm["bk"], ws.data_ptr(), st), "mv2_se_pool")
        _ok(lib.mv2_se_gate(ws.data_ptr(), BF16, T, P, C_, Hd, prm["w1"].data_ptr(), prm["b1"].data_ptr(), prm["w2"].data_ptr(),
                            prm["b2"].data_ptr(), gates.data_ptr(), st), "mv2_se_gate")
        _ok(lib.mv2_gate_residual(y.data_ptr(), x.data_ptr(), gates.data_ptr(), out.data_ptr(), BF16, T, P, C_, st),
            "mv2_gate_residual")
        _ok(lib.mv2_mse(out.data_ptr(), BF16, x.data_ptr(), BF16, out.numel(), mws.data_ptr(), loss.data_ptr(), st), "mv2_mse")
        torch.cuda.synchronize()
        return y, gates, out, loss

    prev = lib.mv2_set_pdl(0)
    try:
        plain = run()
        lib.mv2_set_pdl(1)
        pdl = run()
    finally:
        lib.mv2_set_pdl(prev)
    for a, b in zip(plain, pdl):
        assert torch.equal(a, b)


def test_host_argument_checks():
    """Calls whose arguments the library must refuse before launching anything."""
    lib = _lib()
    st = _st()
    buf = torch.zeros(1 << 12, device="cuda", dtype=torch.float32)
    p = buf.data_ptr()                   # never read: every call passed `p` is refused before it launches anything
    C_, P, Hd = 64, 64, 80
    # se_gate / se_gate_records keep F * Hd hidden floats behind the records, and the workspace reserves F * (C + 16)
    ws = torch.zeros(lib.mv2_se_workspace_bytes(1, P, C_) // 4, device="cuda", dtype=torch.float32)
    w1, w2 = torch.zeros((Hd + 1, C_), device="cuda"), torch.zeros((C_, Hd + 1), device="cuda")
    b1, b2 = torch.zeros(Hd + 1, device="cuda"), torch.zeros(C_, device="cuda")
    gates = torch.empty((1, C_), device="cuda")
    se = (w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(), gates.data_ptr(), st)
    assert lib.mv2_se_gate(ws.data_ptr(), BF16, 1, P, C_, C_ + 17, *se) == E_ARG
    assert b"Hd <= C + 16" in lib.mv2_last_error()
    assert lib.mv2_se_gate_records(ws.data_ptr(), 2, 1, C_, C_ + 17, *se) == E_ARG
    assert lib.mv2_se_gate(ws.data_ptr(), BF16, 1, P, C_, C_ + 16, *se) == 0      # the largest legal hidden width
    assert lib.mv2_se_gate_records(ws.data_ptr(), 2, 1, C_, C_ + 16, *se) == 0
    torch.cuda.synchronize()
    assert lib.mv2_lfq_entropy_partials(p, 8, 13, 1, 100.0, p, p, st) == E_ARG            # d > 12
    lv = (C.c_int32 * 3)(8, 1, 5)
    assert lib.mv2_fsq_forward(p, F32, 8, 16, 3, 1, lv, p, p, p, p, p, None, None, st) == E_ARG      # a level < 2
    assert lib.mv2_fsq_decode(p, 0, 8, 16, 3, 1, lv, p, p, p, F32, st) == E_ARG
    assert lib.mv2_pad_cl(p, p, F32, 1, 3, 4, 5, 2, 1, 1, 5, 1, st) == E_ARG              # reflect pad == W
    assert lib.mv2_pad_cl(p, p, F32, 1, 3, 4, 5, 2, 3, 1, 1, 1, st) == E_ARG              # reflect pad == T
    assert lib.mv2_pad_cl(p, p, F32, 1, 3, 4, 5, 2, 1, 1, 6, 3, st) == E_ARG              # circular pad > W
