"""Which kernel Engine.conv runs for each conv call of the benchmark's README and cfg4 tokenize + decode, and at the edges of
the choice (fp32, use_tc off, tc_variant "tap", a token shift, a feed-forward of width C % 16 != 0, streaming histories,
conv_out where its rule and the slab kernel's differ).  Engine.conv_kernel asks the library's host-side shape queries
only, so this runs without a GPU."""
import types

import pytest
import torch

from magvit2_pytorch_b200._lib import ACT_ELU, ACT_SILU, SHUFFLE_SPACE, SHUFFLE_TIME
from magvit2_pytorch_b200.engine import (Engine, pack_conv, pack_conv_down_space, pack_conv_in_kwpack, pack_ff)

BF, F32 = torch.bfloat16, torch.float32
RES = torch.empty(1)          # stands for a residual operand: the queries only test whether one is given


def _conv(Co, Ci, *k, dt=BF, down=False, **kw):
    w = torch.zeros((Co, Ci) + k)
    pk = pack_conv(w, torch.zeros(Co), dt, **kw)
    if down:
        pack_conv_down_space(pk, w)
    return pk


def _kwpack(Co, Ci, k):
    return pack_conv_in_kwpack(torch.zeros((Co, Ci) + k), torch.zeros(Co))


def _ff(C, I, dt=BF):
    return pack_ff(torch.zeros(2 * I, C, 1, 1, 1), torch.zeros(2 * I), torch.zeros(C, I, 1, 1, 1), torch.zeros(C), dt)


# a case: name, x shape, pack, conv keywords, the kernel it runs (bf16, use_tc on, tc_variant "auto")
def _k333(B, T, HW, C):
    return (f"k333 C{C} {HW}x{HW} T{T}", (B, T, HW, HW, C), lambda: _conv(C, C, 3, 3, 3), dict(act=ACT_ELU), "slab")


def _time_down(B, T, HW, Ci, Co):
    return (f"time down {Ci}->{Co} {HW}x{HW}", (B, T, HW, HW, Ci), lambda: _conv(Co, Ci, 3, k=(3, 1, 1)),
            dict(stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=((T - 1) // 2 + 1, HW, HW)), "slab")


def _space_down(B, T, HW, Ci, Co, down):
    return (f"space down {Ci}->{Co} {HW}x{HW}" + (" down pack" if down else ""), (B, T, HW, HW, Ci),
            lambda: _conv(Co, Ci, 3, 3, down=down),
            dict(stride=(1, 2, 2), pad=(0, 1, 1), out_spatial=(T, (HW - 1) // 2 + 1, (HW - 1) // 2 + 1)),
            "down" if down else "tap")


def _space_up(B, T, HW, Ci, Co):
    return (f"space up {Ci}->{Co} {HW}x{HW}", (B, T, HW, HW, Ci), lambda: _conv(4 * Co, Ci, 1, 1, shuffle_q=4),
            dict(act=ACT_SILU, shuffle=SHUFFLE_SPACE), "slab")


def _time_up(B, T, HW, C):
    return (f"time up {C} {HW}x{HW}", (B, T, HW, HW, C), lambda: _conv(2 * C, C, 1, k=(1, 1, 1), shuffle_q=2),
            dict(act=ACT_SILU, shuffle=SHUFFLE_TIME), "slab")


def _linear(name, B, T, HW, Ci, Co, res=False):
    return (f"{name} {Ci}->{Co} {HW}x{HW}", (B, T, HW, HW, Ci), lambda: _conv(Co, Ci, 1, 1, 1),
            dict(res=RES) if res else {}, "slab")


def _readme_like(B, S, dims):
    """The conv calls of one tokenize + decode of the README layer stack: 17 frames + 3 time-padding frames, frame side S,
    stage widths dims = (d0, d1, d2, d3, d_time)."""
    d0, d1, d2, d3, dt = dims
    s1, s2, s3 = S // 2, S // 4, S // 8
    return [
        _k333(B, 20, S, d0), _k333(B, 20, s1, d1), _k333(B, 20, s2, d2), _k333(B, 20, s3, d3),
        _k333(B, 10, s3, dt), _k333(B, 5, s3, dt),
        _space_down(B, 20, S, d0, d1, True), _space_down(B, 20, s1, d1, d2, True), _space_down(B, 20, s2, d2, d3, True),
        _space_down(B, 20, S, d0, d1, False), _space_down(B, 20, s2, d2, d3, False),
        _time_down(B, 20, s3, d3, dt), _time_down(B, 10, s3, dt, dt),
        _space_up(B, 20, s3, d3, d2), _space_up(B, 20, s2, d2, d1), _space_up(B, 20, s1, d1, d0),
        _time_up(B, 5, s3, dt), _time_up(B, 10, s3, dt),
        _linear("linattn q", B, 20, s2, d2, 128), _linear("linattn kv", B, 20, s2, d2, 256),
        _linear("linattn out", B, 20, s2, 128, d2, res=True),
        _linear("attn qkv", B, 20, s3, d3, 768), _linear("attn out", B, 20, s3, 256, d3, res=True),
        _linear("time attn qkv", B, 5, s3, dt, 768), _linear("time attn out", B, 5, s3, 256, dt, res=True),
        (f"conv_in kwpack {S}x{S}", (B, 20, S, S, 32), lambda: _kwpack(d0, 3, (7, 7, 7)), dict(pad=(6, 3, 0)), "slab"),
    ]


README = _readme_like(4, 128, (64, 128, 256, 512, 512))
CFG4 = _readme_like(3, 256, (64, 128, 256, 512, 1024))


def _engine(dtype=BF, use_tc=True, tc_variant="auto"):
    eng = Engine(None)
    eng.dtype, eng.use_tc, eng.tc_variant = dtype, use_tc, tc_variant
    return eng


def _kind(eng, x_shape, pk, hist_T=0, token_shift=False, **kw):
    return eng.conv_kernel(eng._tc_args(x_shape, pk, **kw), pk, hist_T, token_shift)


@pytest.mark.parametrize("workload,cases", [("readme", README), ("cfg4", CFG4)])
def test_benchmark_conv_calls(workload, cases):
    eng = _engine()
    got = {name: _kind(eng, x_shape, make(), **kw) for name, x_shape, make, kw, _ in cases}
    assert got == {name: kind for name, _, _, _, kind in cases}


def _ff_kinds(eng, x_shape, C, I):
    """(fc1 kernel, fc2 kernel) of Engine.feed_forward on x of width C with hidden width I."""
    fc1, fc2 = _ff(C, I, eng.dtype)
    k1 = _kind(eng, x_shape, fc1)
    g_shape = x_shape[:-1] + ((fc1.Co_tc // 2) if k1 != "simt" else I,)
    return k1, _kind(eng, g_shape, fc2, res=RES)


@pytest.mark.parametrize("workload,B,HW,C,I,T,expect", [
    ("readme linattn", 4, 32, 256, 682, 20, ("slab", "slab")), ("readme attn", 4, 16, 512, 1365, 20, ("slab", "slab")),
    ("readme time attn", 4, 16, 512, 1365, 5, ("slab", "slab")),
    ("cfg4 time attn", 3, 32, 1024, 2730, 5, ("tap", "slab"))])      # fc1's 5504 packed columns: over the slab's Co <= 4096
def test_benchmark_feed_forward(workload, B, HW, C, I, T, expect):
    assert _ff_kinds(_engine(), (B, T, HW, HW, C), C, I) == expect


def _conv_out_call(eng, x_shape, pk, tp):
    """(out_cf, kernel) of the conv Engine.conv_out runs on decoder output x (constant padding, no first-frame conv)."""
    calls = []
    eng.model = types.SimpleNamespace(time_padding=tp, separate_first_frame_encoding=False,
                                      conv_out=types.SimpleNamespace(pad_mode="constant"))
    eng._packs = {"conv_out": pk}
    eng.conv = lambda x, pk, **kw: calls.append(kw) or x
    eng.to_channels_first = lambda x, t_crop=0: x
    eng.conv_out(torch.empty(x_shape, device="meta", dtype=eng.dtype))
    (kw,) = calls
    kw.pop("ss")
    return bool(kw.get("out_cf")), _kind(eng, x_shape, pk, **kw)


@pytest.mark.parametrize("name,x_shape,wshape,expect", [
    ("readme", (4, 20, 128, 128, 64), (3, 64, 3, 3, 3), (True, "slab")),
    ("cfg4", (3, 20, 256, 256, 64), (3, 64, 3, 3, 3), (True, "slab")),
    # where conv_out's rule is narrower than the slab kernel's channels-first store: channels-last conv + layout pass
    ("kw 1, Ci 32", (2, 6, 16, 16, 32), (3, 32, 3, 3, 1), (False, "slab")),
    ("kw 5", (2, 6, 16, 16, 64), (3, 64, 3, 5, 5), (False, "simt"))])
def test_conv_out(name, x_shape, wshape, expect):
    eng = _engine()
    pk = _conv(*wshape)
    if not expect[0]:      # the slab kernel itself would take the channels-first call
        assert eng.conv_cf_supported(torch.empty(x_shape, device="meta"), pk, (pk.k[0] - 4, pk.k[1] // 2, pk.k[2] // 2),
                                     (x_shape[1] - 3,) + x_shape[2:4])
    assert _conv_out_call(eng, x_shape, pk, 3) == expect


EDGES = [
    # name, engine switches, x shape, pack, conv keywords, history frames, kernel
    ("fp32 k333", dict(dtype=F32), (1, 5, 16, 16, 64), lambda: _conv(64, 64, 3, 3, 3, dt=F32), dict(act=ACT_ELU), 0, "simt"),
    ("use_tc off k333", dict(use_tc=False), (1, 5, 16, 16, 64), lambda: _conv(64, 64, 3, 3, 3), dict(act=ACT_ELU), 0, "simt"),
    ("tap k333", dict(tc_variant="tap"), (1, 5, 16, 16, 64), lambda: _conv(64, 64, 3, 3, 3), dict(act=ACT_ELU), 0, "tap"),
    ("tap space down pack", dict(tc_variant="tap"), (1, 5, 32, 32, 64), lambda: _conv(128, 64, 3, 3, down=True),
     dict(stride=(1, 2, 2), pad=(0, 1, 1), out_spatial=(5, 16, 16)), 0, "tap"),
    ("tap conv_in kwpack", dict(tc_variant="tap"), (1, 8, 32, 32, 32), lambda: _kwpack(64, 3, (7, 7, 7)),
     dict(pad=(6, 3, 0)), 0, "tap"),
    ("token shift", {}, (1, 5, 16, 16, 64), lambda: _conv(64, 64, 1, 1, 1), dict(token_shift=True), 0, "simt"),
    ("hist slab C64", {}, (2, 3, 16, 16, 64), lambda: _conv(64, 64, 3, 3, 3), {}, 2, "slab"),
    ("hist simt fp32", dict(dtype=F32), (2, 3, 6, 5, 16), lambda: _conv(24, 16, 3, 3, 3, dt=F32), {}, 2, "simt"),
    ("hist tap C32 32x32 in place", dict(tc_variant="tap"), (2, 3, 32, 32, 32), lambda: _conv(32, 32, 3, 3, 3), {}, 2, "tap"),
    ("hist tap C16 8x8 in place", dict(tc_variant="tap"), (2, 3, 8, 8, 16), lambda: _conv(32, 16, 3, 3, 3), {}, 2, "tap"),
    ("hist tap C16 2x2 copied", dict(tc_variant="tap"), (2, 3, 2, 2, 16), lambda: _conv(32, 16, 3, 3, 3), {}, 2, "tap_cat"),
    ("hist tap time down copied", dict(tc_variant="tap"), (2, 2, 8, 8, 16), lambda: _conv(16, 16, 3, k=(3, 1, 1)),
     dict(stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=(1, 8, 8)), 2, "tap_cat"),
]


@pytest.mark.parametrize("name,switches,x_shape,make,kw,hist_T,expect", EDGES, ids=[e[0] for e in EDGES])
def test_edges(name, switches, x_shape, make, kw, hist_T, expect):
    kw = dict(kw)
    token_shift = kw.pop("token_shift", False)
    assert _kind(_engine(**switches), x_shape, make(), hist_T, token_shift, **kw) == expect


@pytest.mark.parametrize("switches,C,I,expect", [
    (dict(), 40, 128, ("simt", "simt")), (dict(), 40, 96, ("simt", "simt")), (dict(use_tc=False), 64, 128, ("simt", "simt")),
    (dict(dtype=F32), 64, 128, ("simt", "simt")), (dict(tc_variant="tap"), 64, 128, ("tap", "tap"))])
def test_feed_forward_edges(switches, C, I, expect):
    """C % 16 != 0 has no wgmma packs: fc1, GEGLU and fc2 run on the CUDA cores, fc2 too when I % 64 == 0."""
    assert _ff_kinds(_engine(**switches), (1, 3, 8, 8, C), C, I) == expect
