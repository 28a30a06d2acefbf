"""Per-launch times of the tensor-core convs of one bench.py step (README config, bf16, 4 clips of 3x17x128x128, the
benchmark's weight and input seeds): tokenize + decode_from_code_indices run --reps times after a warm-up, with device
events around every wgmma conv launch (slab, fused ResidualUnit, SpatialDownsample2x and tap-wise kernels).  Each
repetition is queued behind a GPU spin so the events bracket kernel time rather than host launch gaps.

One row per launch: kernel, shape, slab plan (mw, bn, slab stages; mv2_tc_slab_plan of the conv, for the fused
ResidualUnit that of its 3x3x3 conv), median microseconds and TFLOP/s from the shapes, the bytes the algorithm has to
move (input, weights and output once each, and the residual) and the launch's floor max(FLOP / 989 TFLOP/s, bytes /
3.35 TB/s).  Both rates of the floor are H100 SXM data-sheet figures (dense BF16, HBM3), not measured ones.  Subtotals
split the launches into one-tap ones (1x1x1 convs, Linear layers, the decoder's up-samplers) and the rest.  The card's
name, power limit and the median SM clock during the timed repetitions are printed with the numbers.

    python tools/slab_conv_time.py [--reps 60]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth_data as Wt  # noqa: E402
from bench import README_KW, ClockSampler  # noqa: E402
from magvit2_pytorch_b200 import VideoTokenizer, _lib  # noqa: E402

LAUNCHES = ("mv2_tc_slab_forward", "mv2_tc_ru_forward", "mv2_tc_down_space_forward", "mv2_tc_conv_forward")
KIND = {"mv2_tc_slab_forward": "slab", "mv2_tc_ru_forward": "fused RU", "mv2_tc_down_space_forward": "down space",
        "mv2_tc_conv_forward": "tap"}


class _RecordingLib:
    """The engine's library handle, recording a copy of the arguments of every tensor-core conv launch."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in LAUNCHES:
            return fn

        def launch(args_ref, *rest):          # (hist, stream), or (stream,) for the down-space conv
            a = args_ref._obj
            self.calls.append((name, type(a).from_buffer_copy(a)))
            return fn(args_ref, *rest)
        return launch


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _ru_conv_args(r):
    """The 3x3x3 conv of a fused ResidualUnit launch as slab-conv arguments (for its plan)."""
    a = _lib.TcConvArgs()
    a.x = a.w = a.y = 1
    a.B, a.Ti, a.Hi, a.Wi, a.Ci = r.B, r.T, r.H, r.W, r.C
    a.To, a.Ho, a.Wo, a.Co = r.T, r.H, r.W, r.C
    a.kt, a.kh, a.kw = r.kt, r.kh, r.kw
    a.st = a.sh = a.sw = 1
    a.pt, a.ph, a.pw = r.kt - 1, r.kh // 2, r.kw // 2
    return a


def _describe(lib, name, a):
    if name == "mv2_tc_ru_forward":
        shape = f"{a.B}x{a.T}x{a.H}x{a.W} C{a.C} k{a.kt}{a.kh}{a.kw}+k111"
        a = _ru_conv_args(a)
    else:
        shape = f"{a.B}x{a.To}x{a.Ho}x{a.Wo} {a.Ci}->{a.Co} k{a.kt}{a.kh}{a.kw}" + (f" s{a.st}{a.sh}{a.sw}" if (a.st, a.sh, a.sw) != (1, 1, 1) else "")
    plan = "-"
    if name in ("mv2_tc_slab_forward", "mv2_tc_ru_forward"):
        out = (C.c_int32 * 6)()
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        if lib.mv2_tc_slab_plan(C.byref(a), n_sm, out) == 0:
            plan = f"mw{out[0]} bn{out[1]} ss{out[5]}"
    return shape, plan


PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12        # H100 SXM data sheet: dense BF16 tensor core, HBM3 bandwidth


def _bytes_and_taps(name, a):
    """bf16 bytes a launch has to move at least (input, weights, output once each, and the residual), and its taps"""
    if name == "mv2_tc_ru_forward":                     # x, the 3x3x3 and 1x1x1 weights, y
        taps = a.kt * a.kh * a.kw
        return 2 * (2 * a.B * a.T * a.H * a.W * a.C + (taps + 1) * a.C * a.C), taps + 1
    taps = a.kt * a.kh * a.kw
    out = a.B * a.To * a.Ho * a.Wo * (a.Co // 2 if a.epi_mode == 1 else a.Co)
    n = a.B * a.Ti * a.Hi * a.Wi * a.Ci + taps * a.Ci * a.Co + out + (out if a.res else 0)
    return 2 * n, taps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60, help="timed repetitions of the step (>= 50)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"

    torch.manual_seed(0)
    model = VideoTokenizer(**README_KW)
    Wt.fill_state_dict_(model, 0)
    model = model.cuda().bfloat16().eval()
    video = Wt.synth_video(4, 3, 17, 128, seed=1000).cuda()
    eng = model.engine

    def step():
        codes = model.tokenize(video)
        return model.decode_from_code_indices(codes)

    with torch.no_grad():
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        rec = _RecordingLib(eng.lib)
        eng.lib = rec
        clk = ClockSampler(torch.cuda.current_device())
        clk.start()
        eng._prof = []
        try:
            torch.cuda._sleep(int(100e6))
            step()                                   # records the launch arguments; not timed
            torch.cuda.synchronize()
            calls = list(rec.calls)
            eng._prof = []
            clk.begin()
            for _ in range(args.reps):
                torch.cuda._sleep(int(100e6))        # ~50 ms of GPU spin: the host queues the whole step behind it
                step()
            torch.cuda.synchronize()
            prof = eng._prof
        finally:
            clocks = clk.stop()                      # also ends the nvidia-smi sampler when the timed region fails
            eng._prof = None
            eng.lib = rec._lib

    n = len(calls)
    assert n and len(prof) == n * args.reps, (n, len(prof))
    lib = rec._lib
    print(f"card: {_card()}  (name, power limit, max SM clock)")
    print(f"SM clock during the timed repetitions: median {clocks.get('sm_mhz')} MHz of {clocks.get('sm_max_mhz')} "
          f"({clocks.get('samples')} samples, reasons {clocks.get('reasons')}); {args.reps} repetitions, median per launch")
    print(f"{'#':>3} {'kernel':<10} {'shape':<36} {'plan':<16} {'us':>8} {'TFLOP/s':>8} {'MB':>8} {'floor us':>9}")
    groups = {"one-tap": [0, 0.0, 0.0, 0.0, 0.0], "multi-tap": [0, 0.0, 0.0, 0.0, 0.0]}   # launches, us, FLOP, bytes, floor
    for i, (name, a) in enumerate(calls):
        samples = [prof[r * n + i][0].elapsed_time(prof[r * n + i][1]) * 1e3 for r in range(args.reps)]
        us, flops = statistics.median(samples), prof[i][2]
        nbytes, taps = _bytes_and_taps(name, a)
        floor = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e6
        g = groups["one-tap" if taps == 1 else "multi-tap"]
        for k, v in enumerate((1, us, flops, nbytes, floor)):
            g[k] += v
        shape, plan = _describe(lib, name, a)
        print(f"{i:>3} {KIND[name]:<10} {shape:<36} {plan:<16} {us:>8.1f} {flops / us / 1e6:>8.1f} {nbytes / 1e6:>8.1f} "
              f"{floor:>9.1f}")
    print("floor: max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s), H100 SXM data-sheet rates, not measured ones")
    for label, (cnt, us, fl, nb, floor) in groups.items():
        print(f"{label} launches ({cnt}): {us / 1e3:.3f} ms, {fl / 1e12:.3f} TFLOP, {fl / us / 1e6:.1f} TFLOP/s, "
              f"{nb / 1e9:.3f} GB, floor {floor / 1e3:.3f} ms")
    tot_us = sum(g[1] for g in groups.values())
    tot_fl = sum(g[2] for g in groups.values())
    print(f"all {n} launches: {tot_us / 1e3:.3f} ms, {tot_fl / 1e12:.3f} TFLOP, {tot_fl / tot_us / 1e6:.1f} TFLOP/s")


if __name__ == "__main__":
    main()
