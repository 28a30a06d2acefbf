"""Which kernel Engine.conv runs for each conv of the benchmark's README tokenize + decode in an fp32 model, with torch's TF32
switch on (Engine.tf32: the wgmma kernels in TF32, the same kinds as bf16, the kw-packed conv_in included: 7 x 3 -> 32
fp32 channels, one 128-byte K row) and off (every fp32 conv on the CUDA cores, as before TF32 existed), and the slab plans of
the fp32 shapes: K rows are 128 bytes, 32 fp32 channels, so a TF32 plan has twice the K chunks of the bf16 plan of the
same shape.  Host-side shape queries only: no GPU."""
import ctypes as C

import pytest
import torch

import tests.test_conv_dispatch_cpu as D
from magvit2_pytorch_b200 import _lib
from magvit2_pytorch_b200._lib import MV2_BF16, MV2_TF32, TcConvArgs
from magvit2_pytorch_b200.engine import Engine, pack_conv, pack_conv_down_space, pack_conv_in_kwpack, pack_ff

F32 = torch.float32


def _conv32(Co, Ci, *k, dt=None, down=False, **kw):
    w = torch.zeros((Co, Ci) + k)
    pk = pack_conv(w, torch.zeros(Co), F32, tc=True, **kw)
    if down:
        pack_conv_down_space(pk, w)
    return pk


@pytest.fixture
def tf32_packs(monkeypatch):
    monkeypatch.setattr(D, "_conv", _conv32)
    monkeypatch.setattr(D, "_kwpack", lambda Co, Ci, k: pack_conv_in_kwpack(torch.zeros((Co, Ci) + k), torch.zeros(Co),
                                                                           dtype=F32))


def _engine(tf32):
    eng = Engine(None)
    eng.dtype, eng.tf32 = F32, tf32
    return eng


def _cases():
    return D._readme_like(4, 128, (64, 128, 256, 512, 512))


@pytest.mark.parametrize("tf32", [True, False])
def test_readme_conv_calls(tf32_packs, tf32):
    eng = _engine(tf32)
    for name, x_shape, make, kw, kind in _cases():
        pk = make()
        if name.startswith("conv_in kwpack"):
            assert pk.w_tc.dtype == F32 and pk.Ci_tc * 4 == 128
        got = D._kind(eng, x_shape, pk, **kw)
        assert got == (kind if tf32 else "simt"), (name, got)


@pytest.mark.parametrize("tf32", [True, False])
@pytest.mark.parametrize("B,HW,C,I,T,expect", [(4, 32, 256, 682, 20, ("slab", "slab")), (4, 16, 512, 1365, 20, ("slab", "slab")),
                                               (3, 32, 1024, 2730, 5, ("tap", "slab"))])
def test_feed_forward(tf32, B, HW, C, I, T, expect):
    eng = _engine(tf32)
    fc1, fc2 = pack_ff(torch.zeros(2 * I, C, 1, 1, 1), torch.zeros(2 * I), torch.zeros(C, I, 1, 1, 1), torch.zeros(C), F32,
                       tc=True)
    k1 = D._kind(eng, (B, T, HW, HW, C), fc1)
    k2 = D._kind(eng, (B, T, HW, HW, (fc1.Co_tc // 2) if k1 != "simt" else I), fc2, res=D.RES)
    assert (k1, k2) == (expect if tf32 else ("simt", "simt"))


def test_conv_out_channels_first():
    eng = _engine(True)
    pk = _conv32(3, 64, 3, 3, 3)
    assert eng.conv_cf_supported(torch.empty((4, 20, 128, 128, 64), device="meta"), pk, (-1, 1, 1), (17, 128, 128))


def _plan(Ci, Co, k, dtype, HW=32, T=5, B=1):
    lib = _lib.load()
    a = TcConvArgs(B=B, Ti=T, Hi=HW, Wi=HW, Ci=Ci, To=T, Ho=HW, Wo=HW, Co=Co, kt=k[0], kh=k[1], kw=k[2], st=1, sh=1, sw=1,
                   pt=k[0] - 1, ph=k[1] // 2, pw=k[2] // 2, dtype=dtype)
    out = (C.c_int * 6)()
    assert lib.mv2_tc_slab_plan(C.byref(a), 132, out) == 0, _lib.last_error() if hasattr(_lib, "last_error") else ""
    return list(out)


@pytest.mark.parametrize("Ci,Co,k", [(32, 64, (7, 7, 1)), (64, 64, (3, 3, 3)), (128, 128, (3, 3, 3)), (256, 256, (3, 3, 3)), (512, 512, (3, 3, 3)),
                                     (64, 256, (1, 1, 1)), (32, 64, (1, 1, 1))])
def test_tf32_slab_plans(Ci, Co, k):
    """The fp32 shapes plan on the slab kernel with the tiling (mw, bn, N tiles, tile count) of bf16; only the ring depths
    may be shallower, as each slab and weight stage holds half the channels in the same bytes."""
    mw, bn, ntn, tiles, grid, stages = _plan(Ci, Co, k, MV2_TF32)
    assert [mw, bn, ntn, tiles, grid] == _plan(Ci, Co, k, MV2_BF16)[:5]
    assert stages in (2, 3)


def test_tf32_byte_rules():
    """Channel rules are rules on bytes: the slab kernel needs 64-byte K rows (16 fp32 channels), 128-byte rows for
    in-plane taps along w (32 fp32 channels); the tap-wise kernel 32-byte rows (8 fp32 channels)."""
    lib = _lib.load()

    def args(Ci, k, dtype):
        return TcConvArgs(B=1, Ti=3, Hi=16, Wi=16, Ci=Ci, To=3, Ho=16, Wo=16, Co=64, kt=k[0], kh=k[1], kw=k[2], st=1, sh=1,
                          sw=1, pt=k[0] - 1, ph=k[1] // 2, pw=k[2] // 2, dtype=dtype)
    assert lib.mv2_tc_slab_supported(C.byref(args(16, (1, 1, 1), MV2_TF32)))
    assert not lib.mv2_tc_slab_supported(C.byref(args(8, (1, 1, 1), MV2_TF32)))
    assert lib.mv2_tc_slab_supported(C.byref(args(32, (3, 3, 3), MV2_TF32)))
    assert not lib.mv2_tc_slab_supported(C.byref(args(16, (3, 3, 3), MV2_TF32)))
    assert lib.mv2_tc_conv_supported(C.byref(args(8, (3, 3, 3), MV2_TF32)))
    assert not lib.mv2_tc_conv_supported(C.byref(args(4, (3, 3, 3), MV2_TF32)))
    assert not lib.mv2_tc_conv_supported(C.byref(args(8, (3, 3, 3), MV2_BF16)))
