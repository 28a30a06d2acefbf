"""Host-side plan of the slab conv's narrow N tiles (the video's data gradient through conv_in: channels-first output of
3 channels, 7 x 7 in-plane taps), through the C ABI without a GPU."""
import ctypes as C

import pytest

from magvit2_pytorch_b200 import _lib
from tests.test_slab_plan import N_SM, _args, _plan


def _dgrad_args(B, T, t_pad, H, W, Ci, Co, k):
    """The transposed conv of a causal conv: no leading time pad, the first t_pad output frames not computed, torch's
    (B, C, T, H, W) output."""
    a = _args(B, T + t_pad, H, W, Ci, Co, k)
    a.To = T
    a.pt = -t_pad
    a.out_layout = 1
    return a


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
