"""Streaming at the kernel level, bit for bit: every entry point that continues a clip from carried state against the plain
entry point run on the concatenation.  A conv over chunks with history equals the conv of the whole input restricted to
each chunk's frames; the chunk schedules start with one frame (history shorter than k_t - 1), then take chunks shorter
than the history (the history spans two chunks and is copied) and longer ones (the history is the previous chunk's tail).
Run on the H100 box:  python -m pytest tests -m gpu"""
import ctypes as C

import pytest
import torch

from magvit2_pytorch_b200 import _lib
from magvit2_pytorch_b200.engine import Engine, StreamState, pack_conv, pack_conv_in_kwpack

pytestmark = pytest.mark.gpu


def _engine(dtype, use_tc=True, tc_variant="auto"):
    assert torch.cuda.is_available(), "gpu-marked test without a GPU"
    eng = Engine(None)
    eng.bind(torch.empty(1, device="cuda", dtype=dtype), "test")
    eng.use_tc, eng.tc_variant = use_tc, tc_variant
    return eng


def _rand(*shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda").to(dtype)


def _streamed(fn, x, chunks, out_tdim=1):
    ss, outs, t = StreamState(), [], 0
    for n in chunks:
        outs.append(fn(x[:, t:t + n].contiguous(), ss))
        t += n
    assert t == x.shape[1]
    return torch.cat(outs, dim=out_tdim)


CHUNKS_3 = [1, 1, 3, 2, 1, 4]          # k_t = 3: T_h = 1 < 2, chunk 1 < T_h = 2 (copied history), chunks >= 2 (tail views)

# name, dtype, use_tc, tc_variant, Ci, Co, H, W, kernel counter that must move
CONV3 = [
    ("cuda-core fp32", torch.float32, False, "auto", 16, 24, 6, 5, "simt_conv_calls"),
    ("cuda-core bf16", torch.bfloat16, False, "auto", 16, 24, 6, 5, "simt_conv_calls"),
    ("tap C=16 8x8 (2-frame tiles)", torch.bfloat16, True, "tap", 16, 32, 8, 8, "tc_calls"),
    ("tap C=32 32x32 (1-frame tiles)", torch.bfloat16, True, "tap", 32, 32, 32, 32, "tc_calls"),
    ("tap C=16 2x2 (copied [hist | x])", torch.bfloat16, True, "tap", 16, 32, 2, 2, "tc_calls"),
    ("slab C=64", torch.bfloat16, True, "auto", 64, 64, 16, 16, "slab_calls"),
    ("slab C=128", torch.bfloat16, True, "auto", 128, 64, 16, 24, "slab_calls"),
]


@pytest.mark.parametrize("case", CONV3, ids=[c[0] for c in CONV3])
def test_conv3x3x3_hist(case):
    name, dt, use_tc, variant, Ci, Co, H, W, counter = case
    eng = _engine(dt, use_tc, variant)
    pk = pack_conv(_rand(Co, Ci, 3, 3, 3, dtype=torch.float32, seed=1) * 0.1, _rand(Co, dtype=torch.float32, seed=2), dt)
    x = _rand(2, sum(CHUNKS_3), H, W, Ci, dtype=dt, seed=3)
    ref = eng.conv(x, pk)
    n0 = getattr(eng, counter)
    got = _streamed(lambda c, ss: eng.conv(c, pk, ss=ss), x, CHUNKS_3)
    assert getattr(eng, counter) > n0
    assert torch.equal(got, ref)


@pytest.mark.parametrize("case", [("cuda-core fp32", torch.float32, False, "auto", 16, "simt_conv_calls"),
                                  ("tap C=16 (copied [hist | x], stride 2)", torch.bfloat16, True, "tap", 16, "tc_calls"),
                                  ("slab C=64", torch.bfloat16, True, "auto", 64, "slab_calls")], ids=lambda c: c[0])
def test_time_downsample_hist(case):
    """TimeDownsample2x (front pad 2, stride 2): chunks of even length."""
    name, dt, use_tc, variant, Ci, counter = case
    eng = _engine(dt, use_tc, variant)
    pk = pack_conv(_rand(Ci, Ci, 3, dtype=torch.float32, seed=4) * 0.2, _rand(Ci, dtype=torch.float32, seed=5), dt, k=(3, 1, 1))
    chunks = [2, 2, 4, 2, 6]
    x = _rand(2, sum(chunks), 8, 8, Ci, dtype=dt, seed=6)

    def down(c, ss=None):
        T = c.shape[1]
        return eng.conv(c, pk, stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=((T + 2 - 3) // 2 + 1, 8, 8), ss=ss)
    ref = down(x)
    n0 = getattr(eng, counter)
    got = _streamed(down, x, chunks)
    assert getattr(eng, counter) > n0
    assert torch.equal(got, ref)


def test_conv_in_kwpack_hist():
    """conv_in on the wgmma path: the 7x7x1 conv over the kw-packed 32-channel ingest (64-byte slab rows), k_t = 7."""
    eng = _engine(torch.bfloat16)
    pin = pack_conv_in_kwpack(_rand(64, 3, 7, 7, 7, dtype=torch.float32, seed=7) * 0.05, _rand(64, dtype=torch.float32, seed=8))
    chunks = [1, 2, 5, 3, 1, 8]
    video = _rand(2, 3, sum(chunks), 32, 32, dtype=torch.float32, seed=9)
    x = eng.ingest_kwpack(video, 0, pin)

    def conv_in(c, ss=None):
        return eng.conv(c, pin, pad=(6, 3, 0), ss=ss)
    ref = conv_in(x)
    n0 = eng.slab_calls
    got = _streamed(conv_in, x, chunks)
    assert eng.slab_calls > n0 and torch.equal(got, ref)


def test_conv_out_channels_first_hist():
    """conv_out (C -> 3) writing torch's (B, C, T, H, W) layout from the slab kernel, continued from history."""
    eng = _engine(torch.bfloat16)
    pk = pack_conv(_rand(3, 64, 3, 3, 3, dtype=torch.float32, seed=10) * 0.05, _rand(3, dtype=torch.float32, seed=11), torch.bfloat16)
    x = _rand(2, sum(CHUNKS_3), 16, 16, 64, dtype=torch.bfloat16, seed=12)

    def conv_out(c, ss=None):
        return eng.conv(c, pk, pad=(2, 1, 1), out_spatial=tuple(c.shape[1:4]), out_cf=True, ss=ss)
    ref = conv_out(x)
    got = _streamed(conv_out, x, CHUNKS_3, out_tdim=2)
    assert got.shape == (2, 3, x.shape[1], 16, 16) and torch.equal(got, ref)


def _ru_pack(C_, seed):
    f = lambda *s, k: _rand(*s, dtype=torch.float32, seed=seed + k)   # noqa: E731
    hid = max(C_ // 2, 16)
    return dict(conv3=pack_conv(f(C_, C_, 3, 3, 3, k=0) * 0.03, f(C_, k=1), torch.bfloat16),
                conv1=pack_conv(f(C_, C_, 1, 1, 1, k=2) * 0.1, f(C_, k=3), torch.bfloat16),
                wk=f(C_, k=4), bk=0.1, w1=f(hid, C_, k=5) * 0.1, b1=f(hid, k=6), w2=f(C_, hid, k=7) * 0.1, b2=f(C_, k=8),
                hidden=hid)


@pytest.mark.parametrize("C_", [64, 128])
def test_fused_residual_unit_hist(C_):
    """The fused ResidualUnit (3x3x3 + ELU + 1x1x1 + ELU + SE pool records in one launch), its SE gates and residual."""
    eng = _engine(torch.bfloat16)
    p = _ru_pack(C_, 20)
    x = _rand(2, sum(CHUNKS_3), 16, 16, C_, dtype=torch.bfloat16, seed=13)
    ref = eng.residual_unit(x, p)
    n0 = eng.fused_ru_calls
    got = _streamed(lambda c, ss: eng.residual_unit(c, p, ss), x, CHUNKS_3)
    assert eng.fused_ru_calls > n0 and torch.equal(got, ref)


@pytest.mark.parametrize("dt,C_", [(torch.float32, 24), (torch.bfloat16, 24), (torch.bfloat16, 64), (torch.bfloat16, 1024)])
def test_rmsnorm_prev(dt, C_):
    """mv2_rmsnorm_prev: the token shift of a continued chunk reads the previous chunk's last frame."""
    eng = _engine(dt)
    gamma = _rand(C_, dtype=torch.float32, seed=14)
    x = _rand(2, 7, 3, 5, C_, dtype=dt, seed=15)
    ref = eng.rmsnorm(x, gamma, token_shift=True)
    got = _streamed(lambda c, ss: eng.rmsnorm(c, gamma, token_shift=True, ss=ss), x, [1, 1, 3, 2])
    assert torch.equal(got, ref)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("L,q0", [(5, 0), (5, 4), (8, 3), (13, 9), (13, 12), (40, 17), (40, 33)])
def test_attention_tail(dt, L, q0):
    """mv2_attention_tail over a K/V cache equals rows [q0, L) of the whole causal call (L <= 8: the short-sequence
    kernel in bf16; L > 8: the general kernel)."""
    lib = _lib.load()
    code = _lib.MV2_F32 if dt == torch.float32 else _lib.MV2_BF16
    B, HW, heads, dh, n_mem = 2, 12, 8, 32, 4
    HD = heads * dh
    qkv = _rand(B, L, HW, 3 * HD, dtype=dt, seed=16)
    mem = _rand(2, heads, n_mem, dh, dtype=torch.float32, seed=17)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    full = torch.empty((B, L, HW, HD), device="cuda", dtype=dt)
    a = _lib.AttnArgs(qkv=qkv.data_ptr(), out=full.data_ptr(), mem_kv=mem.data_ptr(), dtype=code, heads=heads, dim_head=dh,
                      n_mem=n_mem, causal=1, n_outer=B, n_inner=HW, L=L, outer_stride=L * HW, inner_stride=1, tok_stride=HW)
    _lib.check(lib.mv2_attention(C.byref(a), st), "mv2_attention")
    cap = L + 3                                            # a cache with spare capacity, as the engine keeps it
    kv = torch.zeros((B, cap, HW, 2 * HD), device="cuda", dtype=dt)
    kv[:, :L] = qkv[..., HD:]
    q = qkv[:, q0:].contiguous()
    out = torch.empty((B, L - q0, HW, HD), device="cuda", dtype=dt)
    t = _lib.AttnArgs(qkv=kv.data_ptr(), out=None, mem_kv=mem.data_ptr(), dtype=code, heads=heads, dim_head=dh, n_mem=n_mem,
                      causal=1, n_outer=B, n_inner=HW, L=L, outer_stride=cap * HW, inner_stride=1, tok_stride=HW)
    _lib.check(lib.mv2_attention_tail(C.byref(t), q.data_ptr(), (L - q0) * HW, q0, out.data_ptr(), (L - q0) * HW, st),
               "mv2_attention_tail")
    assert torch.equal(out, full[:, q0:])


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_gateloop_scan_state(dt):
    """Scanning [a | b] equals scanning a, then b from the carried fp32 state."""
    lib = _lib.load()
    code = _lib.MV2_F32 if dt == torch.float32 else _lib.MV2_BF16
    B, T, P, C_ = 2, 9, 20, 48
    qkva = _rand(B, T, P, 3 * C_, dtype=dt, seed=18)
    res = _rand(B, T, P, C_, dtype=dt, seed=19)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ref = torch.empty_like(res)
    _lib.check(lib.mv2_gateloop_scan(qkva.data_ptr(), res.data_ptr(), ref.data_ptr(), code, B, T, P, C_, st), "scan")
    state = torch.zeros((B, P, C_), device="cuda", dtype=torch.float32)
    outs = []
    for t0, n in ((0, 1), (1, 3), (4, 5)):
        a, r = qkva[:, t0:t0 + n].contiguous(), res[:, t0:t0 + n].contiguous()
        o = torch.empty_like(r)
        _lib.check(lib.mv2_gateloop_scan_state(a.data_ptr(), r.data_ptr(), o.data_ptr(), code, B, n, P, C_, state.data_ptr(), st),
                   "scan_state")
        outs.append(o)
    assert torch.equal(torch.cat(outs, 1), ref)
