"""The slab conv's launch plan at every slab-conv shape of the README step (bench.py: tokenize + decode of 4 clips of
17 x 128 x 128 at the README config), through the C ABI without a GPU.  The epilogue's shared memory (output and
residual tiles, or accumulator staging) lies inside the same span for every flavour but the fused ResidualUnit, so
these tuples do not depend on how the epilogue uses it."""
import ctypes as C

import pytest

from magvit2_pytorch_b200 import _lib

N_SM = 132

# ((B, T, H, W, Ci, Co, (kt, kh, kw)), (mw, bn, n_tiles_n, total tiles, grid, slab stages))
README_STEP_PLANS = [
    ((4, 10, 16, 16, 512, 1024, (1, 1, 1)), (1, 128, 8, 640, 132, 3)),
    ((4, 10, 16, 16, 512, 512, (1, 1, 1)), (1, 128, 4, 320, 132, 3)),
    ((4, 10, 16, 16, 512, 512, (3, 1, 1)), (1, 128, 4, 320, 132, 3)),
    ((4, 10, 16, 16, 512, 512, (3, 3, 3)), (1, 128, 4, 320, 132, 3)),
    ((4, 17, 128, 128, 64, 3, (3, 3, 3)), (2, 32, 1, 4352, 132, 3)),
    ((4, 20, 128, 128, 32, 64, (7, 7, 1)), (2, 64, 1, 5120, 132, 2)),
    ((4, 20, 16, 16, 1408, 512, (1, 1, 1)), (1, 128, 4, 640, 132, 3)),
    ((4, 20, 16, 16, 256, 512, (1, 1, 1)), (1, 128, 4, 640, 132, 3)),
    ((4, 20, 16, 16, 512, 1024, (1, 1, 1)), (1, 128, 8, 1280, 132, 3)),
    ((4, 20, 16, 16, 512, 2816, (1, 1, 1)), (1, 128, 22, 3520, 132, 3)),
    ((4, 20, 16, 16, 512, 512, (1, 1, 1)), (1, 128, 4, 640, 132, 3)),
    ((4, 20, 16, 16, 512, 512, (3, 3, 3)), (1, 128, 4, 640, 132, 3)),
    ((4, 20, 16, 16, 512, 768, (1, 1, 1)), (1, 128, 6, 960, 132, 3)),
    ((4, 20, 32, 32, 128, 256, (1, 1, 1)), (1, 128, 2, 1280, 132, 3)),
    ((4, 20, 32, 32, 256, 128, (1, 1, 1)), (1, 128, 1, 640, 132, 3)),
    ((4, 20, 32, 32, 256, 1408, (1, 1, 1)), (1, 128, 11, 7040, 132, 3)),
    ((4, 20, 32, 32, 256, 256, (1, 1, 1)), (1, 128, 2, 1280, 132, 3)),
    ((4, 20, 32, 32, 256, 256, (3, 3, 3)), (1, 128, 2, 1280, 132, 3)),
    ((4, 20, 32, 32, 256, 512, (1, 1, 1)), (1, 128, 4, 2560, 132, 3)),
    ((4, 20, 32, 32, 704, 256, (1, 1, 1)), (1, 128, 2, 1280, 132, 3)),
    ((4, 20, 64, 64, 128, 256, (1, 1, 1)), (1, 128, 2, 5120, 132, 3)),
    ((4, 5, 16, 16, 1408, 512, (1, 1, 1)), (1, 128, 4, 160, 132, 3)),
    ((4, 5, 16, 16, 256, 512, (1, 1, 1)), (1, 128, 4, 160, 132, 3)),
    ((4, 5, 16, 16, 512, 1024, (1, 1, 1)), (1, 128, 8, 320, 132, 3)),
    ((4, 5, 16, 16, 512, 2816, (1, 1, 1)), (1, 128, 22, 880, 132, 3)),
    ((4, 5, 16, 16, 512, 512, (1, 1, 1)), (1, 128, 4, 160, 132, 3)),
    ((4, 5, 16, 16, 512, 512, (3, 1, 1)), (1, 128, 4, 160, 132, 3)),
    ((4, 5, 16, 16, 512, 512, (3, 3, 3)), (1, 128, 4, 160, 132, 3)),
    ((4, 5, 16, 16, 512, 768, (1, 1, 1)), (1, 128, 6, 240, 132, 3)),
]


@pytest.mark.parametrize("shape,plan", README_STEP_PLANS)
def test_readme_step_plan(shape, plan):
    B, T, H, W, Ci, Co, (kt, kh, kw) = shape
    a = _lib.TcConvArgs()
    a.x = a.w = a.y = 1                      # never dereferenced by the planning call
    a.B, a.Ti, a.Hi, a.Wi, a.Ci = B, T, H, W, Ci
    a.To, a.Ho, a.Wo, a.Co = T, H, W, Co
    a.kt, a.kh, a.kw = kt, kh, kw
    a.st = a.sh = a.sw = 1
    a.pt, a.ph, a.pw = kt - 1, kh // 2, kw // 2
    a.out_layout = 1 if Co % 8 else 0        # conv_out: 3 channels, channels-first
    out = (C.c_int32 * 6)()
    lib = _lib.load()
    assert lib.mv2_tc_slab_plan(C.byref(a), N_SM, out) == 0, lib.mv2_last_error()
    assert tuple(out) == plan
