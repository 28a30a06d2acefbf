"""The attention cores of csrc/simt_ops.cu, one C ABI call at a time, against float64 references at their tile, mask and
dispatch edges: mv2_attention (softmax attention with prepended memory key/values) and mv2_linear_attention (the Taylor
linear attention, dim_head 8), both activation dtypes.

Dispatch (mv2_attention / mv2_linear_attention; _attn_kernel / _linattn_kernels restate it and every call asserts it):
  * attention_kernel<T, D / 32>: fp32 always; bf16 when causal with L > 8, non-causal with 9 <= L < 64, D = 96, or
    n_mem > 8 with L <= 8.  32 queries per block, 32-key tiles, online softmax with expf.
  * attention_small_kernel<D / 32>: bf16, L <= 8, n_mem <= 8, D 32 / 64; one warp per (sequence, head) with __expf; the
    last block is partial when n_seq * heads % 8 != 0.
  * attention_mma_kernel<D>: bf16, non-causal, L >= 64, D 32 / 64; 128-query blocks, 64-key tiles prefetched one ahead,
    P rounded to bf16 for P V while the denominator l sums the fp32 P, memory key/values rounded to bf16 on load.
  * linear, fp32: linattn_reduce_kernel<float> + linattn_apply_kernel<float> (256-token chunks; the apply kernel sums the
    chunk partials itself).  bf16: linattn_reduce_mma_kernel (128-token staging batches) + linattn_finalize_kernel +
    linattn_apply_mma_kernel (64-token sub-blocks, 4 per block), phi and S carried as bf16 hi + lo pairs.
  * unreachable: linattn_reduce_kernel<bf16> / linattn_apply_kernel<bf16>, whose guard (heads * 8) % 8 == 0 always holds.
test_dispatch_under_profiler runs every case under torch.profiler and checks that each call launched exactly the named
instance(s) and that every reachable instance above was launched.

Guards on every call.  Outputs and the linear-attention workspace (passed at exactly mv2_linattn_workspace_bytes) are
NaN-filled between sentinel blocks (the _Guard allocator of tests/test_conv_forward_gpu.py): an element never written, or a
workspace partial read but never written, poisons the result, and a store outside fails the sentinel check; output rows the
call does not address must stay NaN.  The qkv / q / kv inputs and mem_kv sit in NaN-filled buffers whose rows outside the
addressed tokens (before, after and, in the strided cases, between sequences: outer_stride larger than needed) are NaN, so a
row read that must not be read yields NaN (0 * NaN = NaN in the P V sum).  Every pointer is 16-byte aligned: the MMA paths
load 16 bytes at a time and nothing checks the alignment, a precondition these tests do not probe.

Operands.  Every q / k / v value is bf16-representable, so kernel and reference see the same operands; mem_kv is too, as
pack_attn rounds it to the model dtype (asserted on a bf16 model's pack).  Softmax (_attn_operands): for every query a key at
its last valid position (n_mem + L - 1, or n_mem + i under the causal mask) carries >= 10% of its softmax weight (asserted),
and key 0 holds a smaller maximum (score 2 below it) in the first tile, so the online rescale across tiles matters.  One case
per kernel has scores over about [-75, 60], where exp underflows for most keys.  Taylor (_taylor_operands): the tokens of
the last 128-token staging batch have |k| 16x the others', the last token 32x, so they dominate S through the quadratic
features.

Softmax bound (_softmax64).  w_j is the exact softmax weight, o = sum_j w_j v_j, u = 2^-24, gamma_c(n) = c n u / (1 - c n u)
(Higham, Accuracy and Stability, 3.1 / 3.5; c = 1 for round-to-nearest fma chains, c = 2 for mma.sync, whose fp32 adds may
truncate, see tests/test_conv_grad_gpu.py).  The kernel's p_j = exp(s^_j - m) for its own running max m: m and the corr
factors multiply numerator and denominator alike and cancel, so what matters is the relative error eps_j of each p_j:
  * score: gamma_c(D) scale A_j, A_j = sum_d |q_d k_jd|, plus the roundings after the dot product, each relative to at most
    scale A_j: rsqrtf (2 ulp = 2^-22, CUDA Programming Guide, single-precision math table), the scale product (u), and in
    the MMA kernel fp32(log2 e) and its product with rsqrtf (2 u): (gamma_c(D) + 2^-22 + 4u) scale A_j;
  * the argument s^_j - m: one rounding, u (s_max - s_j);
  * the exponential: expf and exp2f 2 ulp (2^-22 relative); __expf 2 + floor(1.173 |x|) ulp (CUDA Programming Guide,
    intrinsic functions table), taken as (3 + 1.173 x) 2^-23 with x = s_max - s_j;
  eps_j = expm1 of their sum.  Propagated through the normalised weights: sum_j w_j eps_j (|v_je| + |o_e|).
  * sums: p V and l over the M = n_mem + L keys, plus one rounding per tile rescale of o and of l (n_t tiles) and the
    5-level warp reductions: gamma_c(M + n_t + 5) (sum_j w_j |v_je| + |o_e|);
  * MMA kernel: P rounded to bf16 (u_bf16 = 2^-8, 8 significant bits) in the numerator only: 2^-8 sum_j w_j |v_je|;
  * final step: 1 / l (IEEE division) and the product: 2u |o_e|;
  * underflow: a p or corr below 2^-126 (relative to the running max, so to l >= 1) flushes: M 2^-125 (max|v_e| + |o_e|);
  the whole multiplied by 1 + 2^-6 for the products of these relative errors (each below 2^-8 of the larger), plus half an
  ulp of the output dtype (_check).
Taylor bound (_taylor64).  phi(x) = [1, x, x (x) x / sqrt 2]; num_e = sum_f phi_f(q') S_fe, den = the same with v_e = 1,
q' = q / sqrt 8.  With Mabs_e = sum_f |phi_f(q')| sum_n |phi_f(k_n)| |[v_n, 1]_e| (float64), |d num_e| <= delta Mabs_e,
|d den| <= delta Mabs_8 and |d o_e| <= (|d num_e| + |o_e| |d den|) / (den - |d den|) + u |o_e| (the division), den >= L / 2
since 1 + x + x^2 / 2 >= 1/2.  delta adds:
  * phi(q'): rsqrtf(8) 2^-22 and the product u per factor, two factors, fp32(1/sqrt 2) u and two products 2u: 2^-21 + 5u;
  * phi(k): k_i k_j of bf16 operands is exact in fp32; fp32(1/sqrt 2) u and the product u: 2u;
  * fp32 path: the token sum, depth <= 256 within a chunk plus n_chunks across chunks, gamma_1(256 + n_chunks); the feature
    sum gamma_1(73);
  * bf16 path: a = hi + lo with hi = bf16(a): |a - hi| <= 2^-8 |a| and, being below a's bf16 half ulp, rounds to lo within
    2^-17 |a|; that for phi(k), phi(q') and S (3 2^-17), plus the omitted lo lo term (2^-8 (1 + 2^-8))^2; the reduce's
    tensor-core sum over hi and lo products of <= 256 tokens and 4 warps gamma_2(516), the finalize sum gamma_1(n_chunks),
    the apply's 3 MMAs over 80 features gamma_2(240);
  the whole times 1 + 2^-10 for second-order products, plus half an ulp of the output dtype.

Each family shows that its bound rejects a slightly wrong reference.  Softmax: the last key dropped, the memory slots
dropped, the causal mask left-aligned (j <= i) or one key short (j < i + n_mem), scale 1/D, head h's memory taken from head
h + 1, the time layout's token stride one pixel short.  Taylor: the last token dropped, the last chunk dropped, the
quadratic features without 1/sqrt 2, q unscaled, k and v swapped.

Every mv2_attention / mv2_linear_attention call of a bf16 and an fp32 README-config forward and of a bf16 discriminator
forward at 128 px is recorded and checked the same way against float64 restatements of the layout the model implies, which
catches host-side packing errors (strides, n_mem, mem_kv layout, head split) at production shapes."""
import ctypes as C
import math
import re
import types
import weakref
import zlib

import pytest
import torch

from tests.test_conv_forward_gpu import _Guard
from tests.test_conv_grad_gpu import _gamma
from tests.test_simt_ops_gpu import U, _check, _rejects

pytestmark = pytest.mark.gpu

F32, BF16 = 0, 1
DT = {F32: torch.float32, BF16: torch.bfloat16}
E_ARG, E_UNSUPPORTED = -1, -3
DEV = "cuda"
PAD = 7                               # NaN rows in front of and behind every input buffer
U_BF16 = 2.0 ** -8
R_EXP = 2.0 ** -22                    # expf / exp2f / rsqrtf: 2 ulp
LIN_C2 = 0.5 ** 0.5


def _lib():
    from magvit2_pytorch_b200 import _lib as L
    return L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    from magvit2_pytorch_b200._lib import check
    check(rc, what)


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _bf(t):
    return t.to(torch.bfloat16).double()


def _randn(shape, g, scale=1.0):
    return _bf(torch.randn(shape, generator=g, device=DEV, dtype=torch.float64) * scale)


# ------------------------------------------------------------------------------------------------------------------
# dispatch
# ------------------------------------------------------------------------------------------------------------------
def _attn_kernel(code, D, L, n_mem, causal):
    """The kernel instance mv2_attention launches for these arguments."""
    if code == F32:
        return f"attention_kernel<float, {D // 32}>"
    if not causal and L >= 64 and D in (32, 64):
        return f"attention_mma_kernel<{D}>"
    if L <= 8 and n_mem <= 8 and D in (32, 64):
        return f"attention_small_kernel<{D // 32}>"
    return f"attention_kernel<__nv_bfloat16, {D // 32}>"


def _linattn_kernels(code):
    if code == F32:
        return ["linattn_reduce_kernel<float>", "linattn_apply_kernel<float>"]
    return ["linattn_reduce_mma_kernel", "linattn_finalize_kernel", "linattn_apply_mma_kernel"]


REACHABLE = {f"attention_kernel<{t}, {i}>" for t in ("float", "__nv_bfloat16") for i in (1, 2, 3)} | {
    "attention_small_kernel<1>", "attention_small_kernel<2>", "attention_mma_kernel<32>", "attention_mma_kernel<64>",
    *_linattn_kernels(F32), *_linattn_kernels(BF16)}


def _kind(kernel):
    return kernel.split("<")[0].replace("attention_", "").replace("kernel", "").strip("_") or "generic"


KPROP = {   # summation c, keys per tile, exponential, P rounded to bf16 for P V
    "generic": dict(c=1, tile=32, exp="expf", pround=False),
    "small": dict(c=1, tile=16, exp="__expf", pround=False),
    "mma": dict(c=2, tile=64, exp="exp2f", pround=True),
}


# ------------------------------------------------------------------------------------------------------------------
# softmax attention: operands, layout, reference and bound
# ------------------------------------------------------------------------------------------------------------------
def _rows(lay, tok_stride=None):
    """(n_seq, L) qkv / out row of every (sequence, token) of an mv2_attn_args layout."""
    ts = lay["tok_stride"] if tok_stride is None else tok_stride
    s = torch.arange(lay["n_outer"] * lay["n_inner"], device=DEV)
    base = (s // lay["n_inner"]) * lay["outer_stride"] + (s % lay["n_inner"]) * lay["inner_stride"]
    return base[:, None] + torch.arange(lay["L"], device=DEV)[None, :] * ts


def _layout(kind, n_outer, L, HW=1, gap=0):
    if kind == "time":          # Engine.attention's TimeAttention layout, (gap > 0) with unused rows between clips
        return dict(n_outer=n_outer, n_inner=HW, L=L, outer_stride=L * HW + gap, inner_stride=1, tok_stride=HW)
    return dict(n_outer=n_outer, n_inner=1, L=L, outer_stride=L + gap, inner_stride=0, tok_stride=1)


def _attn_operands(n_seq, heads, L, n_mem, D, causal, g, wide=False):
    """q (S,H,L,D), token k / v (S,H,L,D), memory (2,H,n_mem,D), float64 bf16-representable; see the module docstring.
    Coordinate 0 of every query is 2; background keys score ~N(0, 1) (wide: ~N(-30, 15^2)) through the other coordinates;
    key 0 scores sp - 2 and each query's planted key sp = ln(M) + 2 (wide: 60)."""
    scale, a, M = D ** -0.5, 2.0, n_mem + L
    sp = 60.0 if wide else math.log(M) + 2
    sig, off = (15.0, -30.0) if wide else (1.0, 0.0)
    q = _randn((n_seq, heads, L, D), g)
    q[..., 0] = a
    kk = torch.randn((n_seq, heads, L, D), generator=g, device=DEV, dtype=torch.float64) * sig
    mk = torch.randn((heads, n_mem, D), generator=g, device=DEV, dtype=torch.float64) * sig
    kk[..., 0] = mk[..., 0] = off / (scale * a)
    c0 = (sp - 2) / (scale * a)
    if causal and L > 1:        # token i's key scores sp against query i only
        qp = q[..., 1:]
        kk[..., 1:] = qp * (sp / (scale * (qp * qp).sum(-1, keepdim=True)))
        kk[..., 0] = 0
    else:                       # the last key scores sp against every query
        kk[:, :, L - 1] = 0
        kk[:, :, L - 1, 0] = sp / (scale * a)
    if n_mem:                   # the first tile's smaller maximum
        mk[:, 0] = 0
        mk[:, 0, 0] = c0
    else:
        kk[:, :, 0] = 0
        kk[:, :, 0, 0] = c0
    v = _randn((n_seq, heads, L, D), g)
    mv = _randn((heads, n_mem, D), g)
    return q, _bf(kk), v, torch.stack((_bf(mk), mv))


def _softmax64(q, k, v, causal, n_mem, kernel=None, left=False, shift=0, scale=None):
    """float64 softmax attention (oracle.restated.softmax_attention with the memory key/values prepended and the right-aligned
    causal mask, off for L = 1), queries chunked to bound the score blocks.  q (S,H,L,D), k / v (S,H,M,D).
    Returns o, the bound `acc` of `kernel` (None: no bound) and the smallest weight of a query's planted key."""
    S, H, L, D = q.shape
    M = k.shape[2]
    scale = D ** -0.5 if scale is None else scale
    o = torch.empty_like(q)
    acc = torch.empty_like(q) if kernel else None
    i_all = torch.arange(L, device=q.device)[:, None]
    j = torch.arange(M, device=q.device)[None, :]
    masked = causal and L > 1
    planted = (i_all + n_mem) if masked else torch.full_like(i_all, M - 1)
    wmin = math.inf
    lq = max(1, min(L, (1 << 24) // (H * M)))
    if kernel:
        kp = KPROP[_kind(kernel)]
        c, n_t = kp["c"], -(-M // kp["tile"])
        e_s = _gamma(D, c) + R_EXP + 4 * U
        g_sum = _gamma(M + n_t + 5, c)
    for s in range(S):
        for q0 in range(0, L, lq):
            i = i_all[q0:q0 + lq]
            if masked:          # key 0 stays visible, so a shortened mask leaves no query without keys
                valid = (j <= (i if left else i + n_mem) + shift) | (j == 0)
            else:
                valid = torch.ones((i.shape[0], M), dtype=torch.bool, device=q.device)
            qs = q[s, :, q0:q0 + lq]
            sc = torch.einsum("hid,hjd->hij", qs, k[s]) * scale
            sc = sc.masked_fill(~valid, -math.inf)
            w = sc.softmax(dim=-1)
            os_ = torch.einsum("hij,hjd->hid", w, v[s])
            o[s, :, q0:q0 + lq] = os_
            wmin = min(wmin, w.gather(-1, planted[q0:q0 + lq].expand(H, -1, -1)).min().item())
            if not kernel:
                continue
            A = torch.einsum("hid,hjd->hij", qs.abs(), k[s].abs()) * scale
            x = (sc.amax(-1, keepdim=True) - sc).masked_fill(~valid, 0.0)
            e_exp = (3 + 1.173 * x) * 2.0 ** -23 if kp["exp"] == "__expf" else R_EXP
            eps = torch.expm1(e_s * A + U * x + e_exp).masked_fill(~valid, 0.0)
            av, ao = v[s].abs(), os_.abs()
            we = w * eps
            sw = torch.einsum("hij,hjd->hid", w, av)
            t = torch.einsum("hij,hjd->hid", we, av) + we.sum(-1, keepdim=True) * ao
            t = t + g_sum * (sw + ao) + 2 * U * ao + M * 2.0 ** -125 * (av.amax(-2, keepdim=True) + ao)
            if kp["pround"]:
                t = t + U_BF16 * sw
            acc[s, :, q0:q0 + lq] = (1 + 2.0 ** -6) * t
            del A, x, eps, we, sw, t
            del sc, w
    return o, acc, wmin


def _nan_buffer(rows, width, dtype):
    buf = torch.full((rows + 2 * PAD, width), float("nan"), device=DEV, dtype=dtype)
    return buf, buf[PAD:PAD + rows]


class _AttnCall:
    """One mv2_attention call on guarded buffers: qkv with NaN rows outside the addressed tokens, mem_kv inside NaN,
    the output NaN-filled between sentinels."""

    def __init__(self, code, lay, heads, D, n_mem, causal, q, k, v, mem, guard):
        self.code, self.lay, self.heads, self.D, self.n_mem, self.causal = code, lay, heads, D, n_mem, causal
        dt = DT[code]
        HD = heads * D
        rows = _rows(lay)
        n_rows = lay["n_outer"] * lay["outer_stride"]     # every clip, with its trailing gap rows
        _, qkv = _nan_buffer(n_rows, 3 * HD, dt)
        t = torch.stack((q, k, v))                        # (3,S,H,L,D) -> rows (S,L) x (3 H D)
        qkv[rows.reshape(-1)] = t.permute(1, 3, 0, 2, 4).reshape(-1, 3 * HD).to(dt)
        self.qkv64 = qkv.double()
        mbuf = torch.full((mem.numel() + 128,), float("nan"), device=DEV, dtype=torch.float32)
        mbuf[64:64 + mem.numel()] = mem.reshape(-1).float()
        self.mem = mem
        self.out = guard.new((n_rows, HD), dt)
        self.rows = rows
        self.args = dict(qkv=qkv.data_ptr(), out=self.out.data_ptr(), mem_kv=mbuf[64:].data_ptr(), dtype=code, heads=heads,
                         dim_head=D, n_mem=n_mem, causal=int(causal), **lay)
        self._keep = (qkv, mbuf)
        self.kernel = _attn_kernel(code, D, lay["L"], n_mem, causal)

    def run(self):
        from magvit2_pytorch_b200._lib import AttnArgs
        _ok(_lib().mv2_attention(C.byref(AttnArgs(**self.args)), _st()), "mv2_attention")

    def operands(self, tok_stride=None, mem=None):
        """q, k, v (S,H,L / M,D) gathered from the qkv buffer by the layout, memory prepended."""
        S, L, H, D = self.rows.shape[0], self.lay["L"], self.heads, self.D
        t = self.qkv64[_rows(self.lay, tok_stride).reshape(-1)].reshape(S, L, 3, H, D).permute(2, 0, 3, 1, 4)
        mem = self.mem if mem is None else mem
        k = torch.cat((mem[0][None].expand(S, -1, -1, -1), t[1]), dim=2)
        v = torch.cat((mem[1][None].expand(S, -1, -1, -1), t[2]), dim=2)
        return t[0], k, v

    def result(self):
        torch.cuda.synchronize()
        S, L, H, D = self.rows.shape[0], self.lay["L"], self.heads, self.D
        o = self.out.double()
        addressed = torch.zeros(o.shape[0], dtype=torch.bool, device=DEV)
        addressed[self.rows.reshape(-1)] = True
        assert torch.isnan(o[~addressed]).all(), f"{self.kernel}: a store to an output row the call does not address"
        return o[self.rows.reshape(-1)].reshape(S, L, H, D).permute(0, 2, 1, 3)


# name, code, D, heads, layout kind, n_outer, L, HW, gap, n_mem, causal, wide
def _attn_cases():
    cs = []
    nm = (0, 4, 9, 33)
    n = 0
    for D in (32, 64, 96):                      # the generic kernel's edges (and, in bf16, the others where they take them)
        for L in (1, 31, 32, 33, 100):
            for causal in (0, 1):
                cs.append(("gen", D, 2, "seq", 2, L, 1, 3 * (n % 2), nm[n % 4], causal, False))
                n += 1
    cs += [("gen", 32, 3, "time", 2, 33, 5, 4, 9, 1, False), ("gen", 96, 2, "time", 2, 12, 3, 0, 4, 1, False),
           ("gen", 64, 2, "seq", 2, 100, 1, 0, 4, 1, True), ("gen", 32, 2, "seq", 1, 64, 1, 0, 33, 1, False),
           ("gen", 64, 2, "seq", 2, 5, 1, 0, 9, 0, False), ("gen", 32, 2, "seq", 2, 40, 1, 0, 4, 0, False)]
    for n, (L, m) in enumerate([(1, 0), (1, 8), (8, 0), (8, 8), (5, 4), (3, 2), (2, 7), (7, 1), (4, 5)]):
        for causal in (0, 1):                   # the short-sequence kernel: 3 x 3 = 9 warps, the last block partial
            D = (32, 64)[(n + causal) % 2]
            cs.append(("small", D, 3, "time", 1, L, 3, 0, m, causal, False))
    cs += [("small", 32, 2, "seq", 3, 6, 1, 5, 3, 1, False), ("small", 64, 8, "time", 2, 5, 7, 0, 4, 1, True)]
    for n, (L, m, D, H) in enumerate([(64, 0, 32, 1), (65, 4, 64, 8), (127, 60, 32, 8), (128, 70, 64, 1), (129, 4, 32, 8),
                                      (1024, 4, 64, 8), (1024, 70, 32, 1), (189, 4, 64, 1), (187, 4, 32, 8), (64, 60, 64, 8),
                                      (65, 70, 32, 1), (128, 0, 64, 8)]):
        cs.append(("mma", D, H, "seq", 2, L, 1, 3 * (n % 2), m, 0, False))
    cs.append(("mma", 32, 4, "seq", 2, 200, 1, 0, 4, 0, True))
    out = []
    for c in cs:
        for code in (F32, BF16):
            out.append((code,) + c[1:])
    return out


ATTN_CASES = _attn_cases()


def _attn_id(c):
    code, D, H, kind, no, L, HW, gap, m, causal, wide = c
    return (f"{'bf16' if code else 'f32'}-D{D}-h{H}-{kind}{no}x{HW}-L{L}-m{m}-{'c' if causal else 'nc'}"
            f"{'-gap' if gap else ''}{'-wide' if wide else ''}")


def _attn_setup(c, guard):
    code, D, H, kind, no, L, HW, gap, m, causal, wide = c
    lay = _layout(kind, no, L, HW, gap)
    S = lay["n_outer"] * lay["n_inner"]
    q, k, v, mem = _attn_operands(S, H, L, m, D, causal, _gen(*c[1:]), wide)
    return _AttnCall(code, lay, H, D, m, causal, q, k, v, mem, guard)


@pytest.fixture
def guard():
    g = _Guard(types.SimpleNamespace(dtype=torch.float32, device=DEV))
    yield g
    g.check_borders("guarded outputs and workspaces")


@pytest.mark.parametrize("case", ATTN_CASES, ids=[_attn_id(c) for c in ATTN_CASES])
def test_attention(case, guard):
    call = _attn_setup(case, guard)
    call.run()
    out = call.result()
    q, k, v = call.operands()
    ref, acc, wmin = _softmax64(q, k, v, call.causal, call.n_mem, call.kernel)
    assert wmin >= 0.1, f"precondition: a planted key carries only {wmin:.3f} of its query's weight"
    dt = DT[call.code]
    _check(out, ref, dt, acc, call.kernel)
    L, m, H, D = call.lay["L"], call.n_mem, call.heads, call.D
    masked = call.causal and L > 1

    def rej(wrong, what):
        _rejects(out, wrong, dt, acc, f"{call.kernel}: {what}")

    if L + m >= 2:
        keep = torch.arange(L + m - 1, device=DEV)
        if not masked:
            rej(_softmax64(q, k[:, :, keep], v[:, :, keep], False, m)[0], "last key dropped")
    if m:
        rej(_softmax64(q, k[:, :, m:], v[:, :, m:], call.causal, 0)[0], "memory slots dropped")
        if H > 1:
            rej(_softmax64(*call.operands(mem=call.mem.roll(-1, dims=1)), call.causal, m)[0], "head h + 1's memory")
    if masked:
        rej(_softmax64(q, k, v, True, m, shift=-1)[0], "causal mask one key short")
        if m:
            rej(_softmax64(q, k, v, True, m, left=True)[0], "causal mask left-aligned")
    if L + m >= 2:
        rej(_softmax64(q, k, v, call.causal, m, scale=1.0 / D)[0], "scale 1/D")
    if call.lay["n_inner"] > 1 and L > 1:
        rej(_softmax64(*call.operands(tok_stride=call.lay["tok_stride"] - 1), call.causal, m)[0], "token stride one pixel short")


# ------------------------------------------------------------------------------------------------------------------
# Taylor linear attention
# ------------------------------------------------------------------------------------------------------------------
def _taylor_operands(n_seq, heads, L, g):
    """q, k, v (S,H,L,8): q, v ~ N(0, 1); k ~ N(0, 0.25^2), on the last 128-token staging batch N(0, 4^2), last token N(0, 8^2)."""
    q = _randn((n_seq, heads, L, 8), g)
    v = _randn((n_seq, heads, L, 8), g)
    ks = torch.full((L, 1), 0.25, device=DEV, dtype=torch.float64)
    ks[128 * ((L - 1) // 128):] = 4.0
    ks[L - 1] = 8.0
    k = _bf(torch.randn((n_seq, heads, L, 8), generator=g, device=DEV, dtype=torch.float64) * ks)
    return q, k, v


def _phi(z, c2=LIN_C2):
    one = torch.ones_like(z[..., :1])
    return torch.cat((one, z, (z[..., :, None] * z[..., None, :]).flatten(-2) * c2), dim=-1)


def _taylor64(q, k, v, code=None, c2=LIN_C2, qscale=8 ** -0.5, keep=None):
    """float64 Taylor linear attention (oracle.restated.taylor_linear_attention's core) and, for `code`, its bound."""
    L = q.shape[2]
    fq, fk = _phi(q * qscale, c2), _phi(k, c2)
    v1 = torch.cat((v, torch.ones_like(v[..., :1])), dim=-1)
    if keep is not None:
        fk, v1 = fk[:, :, keep], v1[:, :, keep]
    nd = fq @ (fk.transpose(-1, -2) @ v1)
    o = nd[..., :8] / nd[..., 8:].clamp(min=1e-5)
    if code is None:
        return o, None
    nc = -(-L // 256)
    rho = 2.0 ** -21 + 5 * U + 2 * U
    if code == F32:
        delta = rho + _gamma(256 + nc, 1) + _gamma(73, 1)
    else:
        delta = rho + 3 * 2.0 ** -17 + (U_BF16 * (1 + U_BF16)) ** 2 + _gamma(516, 2) + _gamma(nc, 1) + _gamma(240, 2)
    delta *= 1 + 2.0 ** -10
    Mabs = fq.abs() @ (fk.abs().transpose(-1, -2) @ v1.abs())
    dn, dd = delta * Mabs[..., :8], delta * Mabs[..., 8:]
    den = nd[..., 8:]
    assert (den >= L / 2).all()
    return o, (dn + o.abs() * dd) / (den - dd) + U * o.abs()


class _LinCall:
    def __init__(self, code, n_seq, heads, L, q, k, v, guard):
        self.code, self.n_seq, self.heads, self.L = code, n_seq, heads, L
        dt, HD = DT[code], heads * 8
        _, self.q = _nan_buffer(n_seq * L, HD, dt)
        _, self.kv = _nan_buffer(n_seq * L, 2 * HD, dt)
        self.q[:] = q.permute(0, 2, 1, 3).reshape(-1, HD).to(dt)
        self.kv[:] = torch.stack((k, v), dim=2).permute(0, 3, 2, 1, 4).reshape(-1, 2 * HD).to(dt)
        lib = _lib()
        self.ws_bytes = lib.mv2_linattn_workspace_bytes(n_seq, heads, L)
        assert self.ws_bytes % 4 == 0
        self.ws = guard.new((self.ws_bytes // 4,), torch.float32)
        self.out = guard.new((n_seq * L, HD), dt)
        self.kernels = _linattn_kernels(code)

    def run(self):
        _ok(_lib().mv2_linear_attention(self.q.data_ptr(), self.kv.data_ptr(), self.out.data_ptr(), self.code, self.n_seq,
                                        self.L, self.heads, 8, self.ws.data_ptr(), _st()), "mv2_linear_attention")

    def result(self):
        torch.cuda.synchronize()
        return self.out.double().reshape(self.n_seq, self.L, self.heads, 8).permute(0, 2, 1, 3)


LIN_LS = (1, 16, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1024, 4097, 16384)
LIN_CASES = [(code, L, (1, 3, 16)[n % 3] if L != 16384 else 16, (1, 3)[(n // 3) % 2] if L != 16384 else 1)
             for n, L in enumerate(LIN_LS) for code in (F32, BF16)]


def _lin_setup(c, guard):
    code, L, heads, n_seq = c
    q, k, v = _taylor_operands(n_seq, heads, L, _gen(L, heads, n_seq))
    return _LinCall(code, n_seq, heads, L, q, k, v, guard), (q, k, v)


@pytest.mark.parametrize("case", LIN_CASES, ids=[f"{'bf16' if c[0] else 'f32'}-L{c[1]}-h{c[2]}-s{c[3]}" for c in LIN_CASES])
def test_linear_attention(case, guard):
    code, L, heads, n_seq = case
    call, (q, k, v) = _lin_setup(case, guard)
    call.run()
    out = call.result()
    ref, acc = _taylor64(q, k, v, code)
    dt = DT[code]
    _check(out, ref, dt, acc, f"linear attention {call.kernels}")

    def rej(wrong, what):
        _rejects(out, wrong, dt, acc, f"linear attention: {what}")

    if L >= 2:
        rej(_taylor64(q, k, v, keep=torch.arange(L - 1, device=DEV))[0], "last token dropped")
    if L > 256:
        rej(_taylor64(q, k, v, keep=torch.arange(256 * ((L - 1) // 256), device=DEV))[0], "last chunk dropped")
    if L >= 2:          # one token: o = v whatever the weights
        rej(_taylor64(q, k, v, c2=1.0)[0], "quadratic features without 1/sqrt 2")
        rej(_taylor64(q, k, v, qscale=1.0)[0], "q unscaled")
    rej(_taylor64(q, v, k)[0], "k and v swapped")


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
def _short(name):
    base = re.sub(r"^void\s+", "", name).split("(")[0]
    head, _, tail = base.partition("<")
    return (head.split("::")[-1] + (("<" + tail) if tail else "")).replace(" ", "")


def test_dispatch_under_profiler(guard):
    """Every case of test_attention / test_linear_attention under torch.profiler (CUDA activity): each call launches exactly
    the instance(s) the dispatch rule names, and every reachable instance is launched at least once."""
    from torch.profiler import ProfilerActivity, profile
    calls = [_attn_setup(c, guard) for c in ATTN_CASES] + [_lin_setup(c, guard)[0] for c in LIN_CASES]
    want = []
    for cl in calls:
        want += [cl.kernel] if isinstance(cl, _AttnCall) else cl.kernels
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for cl in calls:
            cl.run()
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    got = [_short(e.name) for e in evs if re.search(r"attention|linattn", e.name)]
    assert got == [w.replace(" ", "") for w in want], (len(got), len(want))
    launched = {w for w in want}
    assert launched == REACHABLE, sorted(REACHABLE - launched)
    assert not {n for n in got if "linattn_reduce_kernel<__nv_bfloat16>" in n or "linattn_apply_kernel<__nv_bfloat16>" in n}


# ------------------------------------------------------------------------------------------------------------------
# host argument checks
# ------------------------------------------------------------------------------------------------------------------
def test_host_argument_checks():
    """Calls mv2_attention / mv2_linear_attention must refuse before launching anything: every pointer passed is a
    4-element buffer that no launch could stay inside."""
    from magvit2_pytorch_b200._lib import AttnArgs
    lib = _lib()
    buf = torch.full((4,), float("nan"), device=DEV)
    p = buf.data_ptr()
    good = dict(qkv=p, out=p, mem_kv=p, dtype=BF16, heads=2, dim_head=32, n_mem=4, causal=0, n_outer=1, n_inner=1, L=64,
                outer_stride=64, inner_stride=0, tok_stride=1)
    bad = [dict(dim_head=16), dict(dim_head=33), dict(dim_head=128), dict(heads=0), dict(L=0), dict(n_mem=-1),
           dict(L=32 * 65535 + 1), dict(n_outer=65536, n_inner=32768), dict(mem_kv=None), dict(dtype=2), dict(dtype=F32, L=0)]
    for b in bad:
        assert lib.mv2_attention(C.byref(AttnArgs(**dict(good, **b))), _st()) == E_ARG, b
    assert lib.mv2_linear_attention(p, p, p, BF16, 1, 64, 2, 16, p, _st()) == E_UNSUPPORTED
    assert lib.mv2_linear_attention(p, p, p, F32, 1, 64, 2, 4, p, _st()) == E_UNSUPPORTED
    assert lib.mv2_linear_attention(p, p, p, 2, 1, 64, 2, 8, p, _st()) == E_ARG
    torch.cuda.synchronize()
    assert torch.isnan(buf).all()


# ------------------------------------------------------------------------------------------------------------------
# every attention call of real models
# ------------------------------------------------------------------------------------------------------------------
def _record(monkeypatch, eng):
    """Records every mv2_attention / mv2_linear_attention call of `eng`: the engine-level call it came from (pack, axis,
    input shape), the ABI arguments and copies of the operand and output tensors, found by pointer among the engine's
    allocations and conv outputs."""
    calls, live, ctx = [], {}, {}
    new0, conv0, att0, lin0, lib = eng._new, eng.conv, eng.attention, eng.linear_attention, eng.lib

    def keep(t):
        live[t.data_ptr()] = weakref.ref(t)
        return t

    def tensor(ptr):
        t = live[ptr]()
        assert t is not None and t.data_ptr() == ptr
        return t.clone()

    def attention(x, p, axis):
        ctx.update(p=p, axis=axis, shape=tuple(x.shape))
        return att0(x, p, axis)

    def linear_attention(x, p):
        ctx.update(p=p, axis="linear", shape=tuple(x.shape))
        return lin0(x, p)

    class Lib:
        def __getattr__(self, name):
            return getattr(lib, name)

        def mv2_attention(self, pa, st):
            a = pa._obj
            args = {f: getattr(a, f) for f, _ in a._fields_}
            rc = lib.mv2_attention(pa, st)
            torch.cuda.synchronize()
            calls.append(dict(ctx, op="attn", args=args, qkv=tensor(args["qkv"]), out=tensor(args["out"])))
            return rc

        def mv2_linear_attention(self, q, kv, out, dtype, n_seq, L, heads, dh, ws, st):
            rc = lib.mv2_linear_attention(q, kv, out, dtype, n_seq, L, heads, dh, ws, st)
            torch.cuda.synchronize()
            calls.append(dict(ctx, op="lin", args=dict(dtype=dtype, n_seq=n_seq, L=L, heads=heads, dim_head=dh),
                              q=tensor(q), kv=tensor(kv), out=tensor(out)))
            return rc

    monkeypatch.setattr(eng, "_new", lambda shape, dtype=None: keep(new0(shape, dtype)))
    monkeypatch.setattr(eng, "conv", lambda *a, **kw: keep(conv0(*a, **kw)))
    monkeypatch.setattr(eng, "attention", attention)
    monkeypatch.setattr(eng, "linear_attention", linear_attention)
    monkeypatch.setattr(eng, "lib", Lib())
    return calls


def _check_model_call(c, code, modules=()):
    """One recorded call against float64, its operands read with the layout the model implies: qkv / q / kv channels
    'b n (qkv h d)', time attention over the frames of each pixel (causal), space attention over the pixels of each frame,
    the memory key/values of the module whose parameter the pack carries, the output 'merge heads'."""
    B, T, H, W, _ = c["shape"]
    p, dt = c["p"], DT[code]
    heads, dh = p["heads"], p["dim_head"]
    if c["op"] == "lin":
        q = c["q"].double().reshape(B * T, H * W, heads, dh).permute(0, 2, 1, 3)
        kv = c["kv"].double().reshape(B * T, H * W, 2, heads, dh).permute(2, 0, 3, 1, 4)
        out = c["out"].double().reshape(B * T, H * W, heads, dh).permute(0, 2, 1, 3)
        ref, acc = _taylor64(q, kv[0], kv[1], code)
        _check(out, ref, dt, acc, f"linear attention L={H * W}")
        return
    at = [m for m in modules if m.mem_kv.shape == (2, heads, p["n_mem"], dh)
          and torch.equal(m.mem_kv.detach().to(dt).float(), p["mem_kv"])]
    assert len(at) >= 1, "the pack's mem_kv is no module's memory key/values"
    mem = at[0].mem_kv.detach().to(dt).double()
    t = c["qkv"].double().reshape(B, T, H * W, 3, heads, dh)
    o = c["out"].double().reshape(B, T, H * W, heads, dh)
    if c["axis"] == "time":
        t, o, causal, L = t.permute(3, 0, 2, 4, 1, 5).reshape(3, B * H * W, heads, T, dh), o.permute(0, 2, 3, 1, 4), True, T
    else:
        t, o, causal, L = t.permute(3, 0, 1, 4, 2, 5).reshape(3, B * T, heads, H * W, dh), o.permute(0, 1, 3, 2, 4), False, H * W
    o = o.reshape(t.shape[1:])
    S = t.shape[1]
    k = torch.cat((mem[0][None].expand(S, -1, -1, -1), t[1]), dim=2)
    v = torch.cat((mem[1][None].expand(S, -1, -1, -1), t[2]), dim=2)
    kernel = _attn_kernel(code, dh, L, p["n_mem"], causal)
    ref, acc, _ = _softmax64(t[0], k, v, causal, p["n_mem"], kernel)
    _check(o, ref, dt, acc, f"{c['axis']} attention L={L} ({kernel})")


@pytest.mark.parametrize("code", [BF16, F32], ids=["bf16", "f32"])
def test_readme_forward_attention_calls(monkeypatch, code):
    """A README-config tokenize + decode (1 x 17 x 128 x 128): every attention call against float64, as many as the stages
    imply (one per attend_space / attend_time / linear_attend_space stage on each side)."""
    from magvit2_pytorch_b200.modules import Attention
    from tests.util import README_LAYERS, build_product, golden_video, load_golden
    gold = load_golden("readme")
    assert dict(gold["kwargs"])["layers"] == README_LAYERS
    m = build_product(gold["kwargs"], gold["wseed"]).cuda().to(DT[code])
    eng = m.engine
    calls = _record(monkeypatch, eng)
    with torch.no_grad():
        m.decode_from_code_indices(m.tokenize(golden_video(gold).cuda()))
    torch.cuda.synchronize()
    kinds = [st.kind for st in m.stages]
    want = {op: 2 * sum(k in ks for k in kinds) for op, ks in (("attn", ("attend_space", "attend_time")),
                                                                 ("lin", ("linear_attend_space",)))}
    assert {op: sum(c["op"] == op for c in calls) for op in want} == want
    modules = [a for a in m.modules() if isinstance(a, Attention)]
    if code == BF16:            # pack_attn rounds mem_kv to the model dtype: the MMA kernel's bf16 load is exact
        for pk in (v for v in eng._packs.values() if isinstance(v, dict) and "mem_kv" in v):
            assert torch.equal(pk["mem_kv"], pk["mem_kv"].bfloat16().float())
    for c in calls:
        _check_model_call(c, code, modules)


def test_discriminator_attention_calls(monkeypatch):
    """A bf16 discriminator forward at 128 px: the linear attention of each block (L = 4096 down to 16) against float64."""
    from magvit2_pytorch_b200 import gan
    from magvit2_pytorch_b200.modules import Discriminator
    torch.manual_seed(0)
    d = Discriminator(dim=16, image_size=128, max_dim=128).cuda().bfloat16()
    runner = gan.DiscrRunner(d)
    calls = _record(monkeypatch, runner.eng)
    images = torch.randn((2, 3, 128, 128), generator=_gen("discr"), device=DEV).bfloat16()
    with torch.no_grad():
        runner.forward(images)
    torch.cuda.synchronize()
    assert [c["args"]["L"] for c in calls] == [4096, 1024, 256, 64, 16, 16][:len(d.blocks)]
    assert len(calls) == len(d.blocks) and all(c["args"]["heads"] == 16 for c in calls)
    for c in calls:
        _check_model_call(c, BF16)
