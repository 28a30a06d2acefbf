"""Host-side launch planning of the wgmma slab conv (tiling rule + static tile schedule), through the C ABI without a
GPU: mv2_tc_slab_plan / mv2_tc_slab_tile run the same code mv2_tc_slab_forward and the kernel use."""
import ctypes as C

import pytest

from magvit2_pytorch_b200 import _lib

N_SM = 132


def _args(B, T, H, W, Ci, Co, k=(3, 3, 3), epi_mode=0, shuffle=0):
    kt, kh, kw = k
    a = _lib.TcConvArgs()
    a.x = a.w = a.y = 1                      # never dereferenced by the planning calls
    a.bias = a.res = None
    a.B, a.Ti, a.Hi, a.Wi, a.Ci = B, T, H, W, Ci
    a.To, a.Ho, a.Wo, a.Co = T, H, W, Co
    a.kt, a.kh, a.kw = kt, kh, kw
    a.st = a.sh = a.sw = 1
    a.pt, a.ph, a.pw = kt - 1, kh // 2, kw // 2
    a.act, a.shuffle, a.epi_mode = 0, shuffle, epi_mode
    return a


def _plan(lib, a, n_sm=N_SM):
    out = (C.c_int32 * 6)()
    assert lib.mv2_tc_slab_plan(C.byref(a), n_sm, out) == 0, lib.mv2_last_error()
    return dict(zip(("mw", "bn", "n_tiles_n", "total", "grid", "slab_stages"), out))


def _tiles_of(lib, a, cta, n_sm=N_SM):
    out = (C.c_int32 * 6)()
    k, res = 0, []
    while True:
        assert lib.mv2_tc_slab_tile(C.byref(a), n_sm, cta, k, out) == 0, lib.mv2_last_error()
        if out[0] < 0:
            return res
        res.append(tuple(out))
        k += 1


# README-config conv3 layers (B = 4 clips, 17 + 3 padded frames and the two temporal down-sampling levels)
README_CONV3 = [(4, 20, 128, 128, 64, 64), (4, 20, 64, 64, 128, 128), (4, 20, 32, 32, 256, 256),
                (4, 20, 16, 16, 512, 512), (4, 10, 16, 16, 512, 512), (4, 5, 16, 16, 512, 512)]


@pytest.mark.parametrize("shape", README_CONV3 + [(3, 5, 32, 32, 1024, 1024), (1, 3, 16, 16, 64, 96), (2, 1, 8, 8, 64, 64)])
def test_plan_is_well_formed(shape):
    lib = _lib.load()
    B, T, H, W, Ci, Co = shape
    p = _plan(lib, _args(*shape))
    assert p["mw"] in (1, 2, 4) and p["bn"] in (32, 64, 128)
    assert p["mw"] * p["bn"] <= 128                                   # the M-tile accumulators fit 64 registers per thread
    assert p["slab_stages"] in (2, 3)                               # the ring fits next to the staging at least double-buffered
    assert p["n_tiles_n"] * p["bn"] >= Co > (p["n_tiles_n"] - 1) * p["bn"]   # N tiles cover Co, last one may be ragged
    tiles_per_frame = -(-H // 16) * -(-W // (8 * p["mw"])) * p["n_tiles_n"]
    assert p["total"] == B * T * tiles_per_frame
    assert p["grid"] == min(p["total"], N_SM)


def test_tiling_rule_on_readme_layers():
    lib = _lib.load()
    got = [(_plan(lib, _args(*s))["mw"], _plan(lib, _args(*s))["bn"]) for s in README_CONV3]
    # narrow layers share each weight tile between 2 M-tiles; Co >= 128 takes the widest MMA
    assert got[:3] == [(2, 64), (1, 128), (1, 128)]
    assert got[3:] == [(1, 128)] * 3
    # GEGLU feed-forward: 2 * 1408 packed columns -> 22 tiles of 128
    ff = _plan(lib, _args(4, 20, 16, 16, 512, 2816, k=(1, 1, 1), epi_mode=1))
    assert (ff["mw"], ff["bn"], ff["n_tiles_n"]) == (1, 128, 22)
    # a width with no large power-of-two divisor takes wide tiles with a ragged last one instead of 64-column tiles
    odd = _plan(lib, _args(4, 20, 16, 16, 512, 2752, k=(1, 1, 1), epi_mode=1))
    assert odd["bn"] == 128 and odd["n_tiles_n"] == 22


@pytest.mark.parametrize("shape", [(4, 20, 16, 16, 512, 512), (4, 10, 16, 16, 512, 512), (4, 5, 16, 16, 512, 512),
                                   (2, 3, 40, 24, 64, 64), (1, 1, 16, 16, 64, 64), (4, 20, 32, 32, 256, 256)])
def test_schedule_visits_every_tile_exactly_once(shape):
    lib = _lib.load()
    B, T, H, W, Ci, Co = shape
    a = _args(*shape)
    p = _plan(lib, a)
    seen, coords, per_cta = set(), set(), []
    for cta in range(p["grid"]):
        ts = _tiles_of(lib, a, cta)
        per_cta.append(ts)
        for tile, b, t, h0, w0, n0 in ts:
            assert 0 <= tile < p["total"] and tile not in seen
            seen.add(tile)
            assert 0 <= b < B and 0 <= t < T and h0 % 16 == 0 and h0 < H and w0 % (8 * p["mw"]) == 0 and w0 < W
            assert n0 % p["bn"] == 0 and n0 < Co
            coords.add((b, t, h0, w0, n0))
    assert len(seen) == p["total"] == len(coords)                     # a bijection onto the output tiles
    assert max(len(t) for t in per_cta) - min(len(t) for t in per_cta) <= 1


def test_schedule_is_longest_first_and_balanced():
    """C = 512, T = 20: 640 tiles on 132 CTAs.  Frames t = 0 / 1 see 1 / 2 of the 3 frame taps; the static schedule must
    start every CTA on full-cost tiles and run the cheap tiles in the last, partial wave."""
    lib = _lib.load()
    a = _args(4, 20, 16, 16, 512, 512)
    p = _plan(lib, a)
    assert (p["total"], p["grid"]) == (640, 132)
    cost = lambda t: 3 - max(0, 2 - t)
    loads = []
    for cta in range(p["grid"]):
        ts = _tiles_of(lib, a, cta)
        costs = [cost(t) for _, _, t, _, _, _ in ts]
        assert costs == sorted(costs, reverse=True)                   # each CTA runs its expensive tiles first
        assert costs[0] == 3
        loads.append(sum(costs))
    total = 4 * (18 * 3 + 2 + 1) * 8                                  # clips * per-clip frame cost * tiles per frame
    assert sum(loads) == total
    assert max(loads) == 15                                           # 576 full tiles: no CTA runs more than 5 of them
    assert max(loads) <= -(-total // p["grid"]) + 2


def test_plan_rejects_unsupported_shapes():
    lib = _lib.load()
    a = _args(1, 4, 16, 16, 64, 64)
    a.st = 2
    out = (C.c_int32 * 6)()
    assert lib.mv2_tc_slab_plan(C.byref(a), N_SM, out) < 0
    assert b"unsupported" in lib.mv2_last_error()
