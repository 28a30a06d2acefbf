"""Host-side premises of tests/test_bench_calls_gpu.py (and of tests/test_video_dgrad_gpu.py, which replays and plants
defects the same way), without a GPU:

  * the exact-replay grid: at every GEMM depth K the benchmark's workloads run (README up to 27 x 512 and the GEGLU
    widths, cfg4 up to 27 x 1024) and the video's data gradient runs (init_dim x taps, up to 128 x 343), every product and partial sum of grid operands is a multiple of 2^-8 below 2^14 (22
    significant bits), so an fp32 accumulation is exact in any order, even with an adder that truncates.  Checked by the
    arithmetic and by fp32 sums in shuffled orders against float64;
  * the defect tile choice: the schedule's last tile (mv2_tc_slab_tile) has a predecessor on the same CTA whose output
    region does not overlap it, at the shapes the defects are planted in."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from bench import FRAMES, WORKLOADS
from tests.test_bench_calls_gpu import REPLAY_GRID, last_cta
from tests.test_slab_plan_narrow import VIDEO_DGRAD_SLAB, video_dgrad_args

from magvit2_pytorch_b200 import VideoTokenizer, _lib
from magvit2_pytorch_b200.engine import _round_up

N_SM = 132
# the depths of the video's data gradient: init_dim x the taps of conv_in (7x7x7, 5x5x5, 3x3x3) or of its first-frame conv
VIDEO_DGRAD_DEPTHS = [64 * 343, 128 * 343, 64 * 125, 64 * 49, 64 * 27]


def _gemm_depths(kw):
    """K of every wgmma GEMM of a tokenize + decode: taps x Ci of each conv / linear weight, the down-space pack's 6
    taps x 2 Ci, conv_in's kw-packed 7 x 7 x 32 and fc2's hidden width padded to 64 (pack_ff)."""
    with torch.device("meta"):
        m = VideoTokenizer(**kw)
    ks = {7 * 7 * 32}
    for mod in m.modules():
        if isinstance(mod, (torch.nn.Conv1d, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.Linear)):
            w = mod.weight
            ks.add(w[0].numel())
            if isinstance(mod, torch.nn.Conv2d) and tuple(w.shape[2:]) == (3, 3):
                ks.add(12 * w.shape[1])
            if w.shape[2:].numel() == 1:
                ks.add(_round_up(w.shape[1], 64))
    return m, sorted(ks)


@pytest.mark.parametrize("workload", ["readme", "cfg4", "video_dgrad"])
def test_replay_grid_is_exact_at_every_depth(workload):
    if workload == "video_dgrad":
        ks = VIDEO_DGRAD_DEPTHS
        assert max(ks) == 128 * 343 > 27 * 1024
    else:
        _, ks = _gemm_depths(WORKLOADS[workload]["kw"])
        assert max(ks) == 27 * (1024 if workload == "cfg4" else 512)
    assert_replay_grid_exact(ks)


def assert_replay_grid_exact(ks):
    """REPLAY_GRID operands accumulate exactly in fp32, in any order, at every GEMM depth in ks."""
    (nx, ex), (nw, ew), (nb, eb) = REPLAY_GRID["x"], REPLAY_GRID["w"], REPLAY_GRID["b"]
    # the arithmetic: products are multiples of 2^-(ex + ew); the bias is a multiple of 2^-eb with eb <= ex + ew; the
    # largest partial sum (all products of one sign at their largest, plus the bias) stays below 2^(22 - ex - ew)
    m_ = ex + ew
    assert eb <= m_
    for K in ks:
        worst = K * (nx * 2.0 ** -ex) * (nw * 2.0 ** -ew) + nb * 2.0 ** -eb
        assert worst < 2.0 ** (22 - m_), (K, worst)
    # fp32 sums, in three shuffled orders, of the worst case and of random grid operands equal the float64 sums
    rng = np.random.default_rng(len(ks))
    for K in (max(ks), 27 * 64, 12 * 512):
        worst = np.full(K + 1, nx * nw * 2.0 ** -m_)
        worst[-1] = nb * 2.0 ** -eb
        rand = np.append(rng.integers(-nx, nx + 1, K) * rng.integers(-nw, nw + 1, K) * 2.0 ** -m_,
                         rng.integers(-nb, nb + 1) * 2.0 ** -eb)
        for terms in (worst, -worst, rand):
            exact = terms.sum()
            for _ in range(3):
                order = rng.permutation(K + 1)
                part = np.cumsum(terms[order].astype(np.float32), dtype=np.float32)
                assert part[-1] == exact and np.array_equal(part.astype(np.float64), np.cumsum(terms[order]))


def _args(B, T, H, W, Ci, Co, k, pad, To):
    a = _lib.TcConvArgs()
    a.x = a.w = a.y = 1
    a.bias = a.res = None
    a.B, a.Ti, a.Hi, a.Wi, a.Ci = B, T, H, W, Ci
    a.To, a.Ho, a.Wo, a.Co = To, H, W, Co
    a.kt, a.kh, a.kw = k
    a.st = a.sh = a.sw = 1
    a.pt, a.ph, a.pw = pad
    a.act, a.shuffle, a.epi_mode = 1, 0, 0
    a.out_layout = int(Co % 8 != 0)
    return a


def _defect_shapes(workload):
    """(name, TcConvArgs) of the calls the replay plants its defects in: the fused RU (C = 64 and 128, at the first
    encoder / last decoder resolution), the widest 3x3x3 EPI_PLAIN conv at each frame count, conv_out; for "video_dgrad"
    every slab case of tests/test_video_dgrad_gpu.py."""
    if workload == "video_dgrad":
        return [(name, video_dgrad_args(*shape)) for name, (shape, _) in VIDEO_DGRAD_SLAB.items()]
    kw, clips = WORKLOADS[workload]["kw"], WORKLOADS[workload]["clips"] if workload == "readme" else 1
    s, top = kw["image_size"], kw["max_dim"]
    T = FRAMES + 3
    return [("ru_c64", _args(clips, T, s, s, 64, 64, (3, 3, 3), (2, 1, 1), T)),
            ("ru_c128", _args(clips, T, s // 2, s // 2, 128, 128, (3, 3, 3), (2, 1, 1), T))] + [
            (f"plain_c{c}_T{t}", _args(clips, t, s // 8, s // 8, c, c, (3, 3, 3), (2, 1, 1), t))
            for c, t in ((512, T), (top, T // 2), (top, T // 4))] + [
            ("conv_out", _args(clips, T, s, s, 64, 3, (3, 3, 3), (-1, 1, 1), FRAMES))]


@pytest.mark.parametrize("workload", ["readme", "cfg4", "video_dgrad"])
def test_defect_tile_has_a_disjoint_predecessor(workload):
    lib = _lib.load()
    out = (C.c_int32 * 6)()
    for name, a in _defect_shapes(workload):
        assert lib.mv2_tc_slab_plan(C.byref(a), N_SM, out) == 0, lib.mv2_last_error()
        mw, bn, total, grid = out[0], out[1], out[3], out[4]
        tiles, k = [], 0
        while True:
            assert lib.mv2_tc_slab_tile(C.byref(a), N_SM, last_cta(total, grid), k, out) == 0
            if out[0] < 0:
                break
            tiles.append(tuple(out))
            k += 1
        assert len(tiles) >= 2 and tiles[-1][0] == total - 1, (name, tiles)
        (_, b0, t0, h0, w0, n0), (_, b1, t1, h1, w1, n1) = tiles[-2:]
        overlap = (b0 == b1 and t0 == t1 and abs(h0 - h1) < 16 and abs(w0 - w1) < 8 * mw and abs(n0 - n1) < bn)
        assert not overlap, (name, tiles[-2:])
