"""Host-side plan of the slab conv's narrow N tiles (the video's data gradient through conv_in: channels-first output of
3 channels, 7 x 7 in-plane taps), through the C ABI without a GPU; and the kernel TrainRunner.video_dgrad_packed picks for
every channel count, kernel size and dtype the tokenizer's constructor allows."""
import ctypes as C

import pytest
import torch

from magvit2_pytorch_b200 import _lib
from magvit2_pytorch_b200.engine import Engine
from magvit2_pytorch_b200.train import TrainRunner, transposed_pack
from tests.test_slab_plan import N_SM, _args, _plan

K777, K555, K333, K177 = (7, 7, 7), (5, 5, 5), (3, 3, 3), (1, 7, 7)

# The video-gradient calls tests/test_video_dgrad_gpu.py runs on the slab kernel with more tiles than CTAs:
# name -> ((B, Ti, t_crop, H, W, init_dim, channels, k), (bn, mw, total tiles on 132 SMs)).  Ti counts the time-padding
# frames; the output has Ti - t_crop frames.
VIDEO_DGRAD_SLAB = {
    "readme": ((4, 20, 3, 128, 128, 64, 3, K777), (8, 2, 4352)),
    "readme_c12": ((4, 20, 3, 128, 128, 64, 12, K777), (16, 2, 4352)),
    **{f"c{c}_120": ((2, 20, 3, 120, 120, 64, c, K777), (8 if c <= 8 else 16, 2, 2176)) for c in (1, 2, 7, 9, 15)},
    "first_frame": ((4, 1, 0, 128, 128, 64, 3, K177), (8, 2, 256)),
    "sff_rest": ((4, 16, 0, 128, 128, 64, 3, K777), (8, 2, 4096)),
    "no_first_frame": ((4, 17, 0, 128, 128, 64, 3, K777), (8, 2, 4352)),
    "init_dim128": ((4, 20, 3, 128, 128, 128, 3, K777), (8, 2, 4352)),
    "k555": ((4, 20, 3, 128, 128, 64, 3, K555), (8, 4, 2176)),
    "k333": ((4, 20, 3, 128, 128, 64, 3, K333), (32, 2, 4352)),
    "k333_c17": ((4, 20, 3, 128, 128, 64, 17, K333), (32, 2, 4352)),
}


def _dgrad_args(B, T, t_pad, H, W, Ci, Co, k):
    """The transposed conv of a causal conv: no leading time pad, the first t_pad output frames not computed, torch's
    (B, C, T, H, W) output."""
    a = _args(B, T + t_pad, H, W, Ci, Co, k)
    a.To = T
    a.pt = -t_pad
    a.out_layout = 1
    return a


def video_dgrad_args(B, Ti, t_crop, H, W, init_dim, channels, k):
    """The TcConvArgs of the slab call of a VIDEO_DGRAD_SLAB shape."""
    return _dgrad_args(B, Ti - t_crop, t_crop, H, W, init_dim, channels, k)


@pytest.mark.parametrize("Co,bn", [(3, 8), (1, 8), (12, 16)])
@pytest.mark.parametrize("k", [(7, 7, 7), (1, 7, 7)])
def test_narrow_tile_covers_all_channels_in_one_n_tile(Co, bn, k):
    lib = _lib.load()
    a = _dgrad_args(1, 17, 3, 128, 128, 64, Co, k)
    assert lib.mv2_tc_slab_supported(C.byref(a))
    p = _plan(lib, a)
    assert p["bn"] == bn and p["n_tiles_n"] == 1, p
    tiles_w = -(-128 // (8 * p["mw"]))
    assert p["total"] == 17 * (128 // 16) * tiles_w, p
    assert p["grid"] == min(p["total"], N_SM)


def test_conv_out_keeps_its_plan():
    """conv_out (3x3x3, channels-first, 3 channels) stays on the 32-column tile."""
    lib = _lib.load()
    a = _args(1, 20, 128, 128, 64, 3)
    a.To, a.pt, a.out_layout = 17, 2 - 3, 1
    p = _plan(lib, a)
    assert p["bn"] == 32 and p["n_tiles_n"] == 1, p


def test_wide_channels_first_taps_need_the_narrow_tile():
    lib = _lib.load()
    assert not lib.mv2_tc_slab_supported(C.byref(_dgrad_args(1, 17, 3, 128, 128, 64, 17, (7, 7, 7))))     # > 16 channels
    a = _args(1, 20, 128, 128, 64, 8, (7, 7, 7))                                                 # channels-last 7-wide
    assert not lib.mv2_tc_slab_supported(C.byref(a))


@pytest.mark.parametrize("name", sorted(VIDEO_DGRAD_SLAB))
def test_video_dgrad_gpu_cases_plan(name):
    """Each slab case of the GPU test plans the N tile, macro tile and tile count it is there for, with more tiles than
    CTAs (tests/test_bench_calls_cpu.py shows that the last tile's CTA ran an earlier, disjoint tile)."""
    shape, (bn, mw, total) = VIDEO_DGRAD_SLAB[name]
    p = _plan(_lib.load(), video_dgrad_args(*shape))
    assert (p["bn"], p["mw"], p["total"], p["n_tiles_n"]) == (bn, mw, total, 1), p
    assert p["total"] > p["grid"] == N_SM


# ---------------------------------------------------------------------------------------------------------------------------
# the route of TrainRunner.video_dgrad_packed
# ---------------------------------------------------------------------------------------------------------------------------
# the macro tile of the channels-first slab call at 128^2, per (k, bn): the 5-wide taps' slab fits two stages of a 4-tile
# macro tile beside an 8-column weight tile only
MW_OF = {(K777, 8): 2, (K777, 16): 2, (K555, 8): 4, (K555, 16): 2, (K177, 8): 2, (K177, 16): 2, (K333, 32): 2}


def _route(dtype, channels, k, B=4, Ti=20, t_crop=3, HW=128, init_dim=64):
    """(kernel, channels-first store, t_crop of the layout pass or None, plan) of video_dgrad_packed on an engine whose conv
    records its call: the kernel from Engine.conv_kernel for exactly the arguments video_dgrad_packed passes."""
    eng = Engine(None)
    eng.dtype = dtype
    calls = []

    def conv(g, pk, **kw):
        calls.append(kw)
        To, Ho, Wo = kw["out_spatial"]
        shape = (g.shape[0], pk.Co, To, Ho, Wo) if kw.get("out_cf") else (g.shape[0], To, Ho, Wo, pk.Co)
        return torch.empty(shape, device="meta", dtype=dtype)

    def to_channels_first(x, t_crop=0):
        calls.append(dict(layout=t_crop))
        return x.permute(0, 4, 1, 2, 3)[:, :, t_crop:]

    eng.conv, eng.to_channels_first = conv, to_channels_first
    runner = TrainRunner.__new__(TrainRunner)
    super(TrainRunner, runner).__init__(eng)
    pk = transposed_pack(torch.zeros((init_dim, channels) + k), k, dtype)
    g = torch.empty((B, Ti, HW, HW, init_dim), device="meta", dtype=dtype)
    out = runner.video_dgrad_packed(g, pk, t_crop)
    assert tuple(out.shape) == (B, channels, Ti - t_crop, HW, HW)
    kw, layout = calls[0], (calls[1]["layout"] if len(calls) == 2 else None)
    ta = eng._tc_args(g.shape, pk, pad=kw["pad"], out_spatial=kw["out_spatial"], out_cf=bool(kw.get("out_cf")))
    kind = eng.conv_kernel(ta, pk)
    return kind, bool(kw.get("out_cf")), layout, (_plan(_lib.load(), ta) if kind == "slab" else None)


def _want(dtype, channels, k):
    """The route table: bf16 channels-first on the slab kernel (narrow 8 / 16-column tiles for 7- and 5-wide taps, the
    32-column ragged tile for 3x3x3) unless the channel count is a multiple of 8 or, with wide taps, above 16; then the
    channels-last conv and a layout pass: the slab kernel for 3x3x3, the tap-wise kernel for the 49 taps of the first-frame
    conv, the CUDA-core conv for 343 and 125 taps (more than the tap-wise kernel's 64).  fp32: the CUDA-core conv."""
    if dtype == torch.float32:
        return "simt", False
    if channels % 8 != 0 and (channels <= 16 or k == K333):
        return "slab", True
    return {K333: "slab", K177: "tap"}.get(k, "simt"), False


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("k", [K777, K177, K555, K333], ids=["k777", "k177", "k555", "k333"])
def test_video_dgrad_route(dtype, k):
    Ti, t_crop = (1, 0) if k == K177 else (20, 3)
    for channels in list(range(1, 18)) + [32]:
        kind, cf, layout, plan = _route(dtype, channels, k, Ti=Ti, t_crop=t_crop)
        want_kind, want_cf = _want(dtype, channels, k)
        assert (kind, cf) == (want_kind, want_cf), (channels, kind, cf)
        assert layout == (None if cf else t_crop), (channels, layout)
        if cf:
            bn = 32 if k == K333 else (8 if channels <= 8 else 16)
            mw = MW_OF[k, bn]
            total = 4 * (Ti - t_crop) * 8 * (128 // (8 * mw))
            assert (plan["bn"], plan["mw"], plan["n_tiles_n"], plan["total"]) == (bn, mw, 1, total), (channels, plan)
