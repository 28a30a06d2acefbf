"""IEEE fp32, TF32 and bf16 on the benchmark's step: README config, 4 clips of 3x17x128x128 (the benchmark's weight and input
seeds), tokenize + decode_from_code_indices through StreamLanes(tok, 3) with CUDA graphs on, as bench.py times it.  The
fp32 model runs with torch's TF32 matmul switch off (IEEE: the CUDA-core convs) and on (the TF32 wgmma convs); the three
modes are timed in alternating rounds in one process (--rounds each, --steps steps per round after a warm-up that
captures every lane's graphs), so drift of the shared card's clocks hits them alike.  Then the per-launch times of the TF32
tensor-core convs of one step (device events around every launch, each repetition queued behind a GPU spin) with their
TFLOP/s against the H100 SXM data sheet's 495 dense TF32 TFLOP/s, and the device time of every kernel of the step by name
(torch.profiler) for IEEE fp32 and TF32.  The card's name, power limit and the median SM clock during the timed rounds are
printed with the numbers.

    python tools/tf32_time.py [--rounds 5] [--steps 30] [--reps 10]
"""
from __future__ import annotations

import argparse
import contextlib
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth_data as Wt  # noqa: E402
from bench import ClockSampler  # noqa: E402
from magvit2_pytorch_b200 import StreamLanes  # noqa: E402
from tools.f16_time import CLIPS, FRAMES, _kernel_times, _model, _per_launch, _round, _step  # noqa: E402
from tools.slab_conv_time import KIND, _card, _describe  # noqa: E402

TF32_PEAK = 495e12          # H100 SXM5 data sheet, dense TF32 tensor-core rate


@contextlib.contextmanager
def _precision(mode):
    """torch's fp32 matmul switch for a mode: "tf32" for TF32, "ieee" otherwise; restored afterwards."""
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if mode == "tf32" else "ieee"
    try:
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating timed rounds per mode (>= 3)")
    ap.add_argument("--steps", type=int, default=30, help="steps per round")
    ap.add_argument("--reps", type=int, default=10, help="repetitions of the per-launch and per-kernel timings")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert args.rounds >= 3

    modes = ("fp32", "tf32", "bf16")
    models = {k: _model(torch.bfloat16 if k == "bf16" else torch.float32) for k in modes}
    batches = {k: [Wt.synth_video(CLIPS, 3, FRAMES, 128, seed=1000 + i).cuda().to(m.dtype) for i in range(2)]
               for k, m in models.items()}
    lanes = {k: StreamLanes(m, 3) for k, m in models.items()}
    steps = {k: _step(m) for k, m in models.items()}
    with torch.no_grad():
        for k in modes:
            with _precision(k):
                for i in range(9):                        # every lane: plain call, graph capture, first replay
                    lanes[k].run(steps[k], batches[k][i % 2])
                lanes[k].join()
        torch.cuda.synchronize()
        clk = ClockSampler(torch.cuda.current_device())
        clk.start()
        clk.begin()
        times = {k: [] for k in modes}
        try:
            for _ in range(args.rounds):
                for k in modes:
                    with _precision(k):
                        times[k].append(_round(lanes[k], steps[k], batches[k], args.steps))
        finally:
            clocks = clk.stop()
        with _precision("tf32"):
            calls, us, flops = _per_launch(models["tf32"], batches["tf32"][0], args.reps)
            k_tf32 = _kernel_times(models["tf32"], batches["tf32"][0], args.reps)
        with _precision("fp32"):
            k_fp32 = _kernel_times(models["fp32"], batches["fp32"][0], args.reps)

    print(f"card: {_card()}  (name, power limit, max SM clock)")
    print(f"SM clock during the timed rounds: median {clocks.get('sm_mhz')} MHz of {clocks.get('sm_max_mhz')} "
          f"({clocks.get('samples')} samples, reasons {clocks.get('reasons')})")
    frames = CLIPS * FRAMES
    for k in modes:
        ms = statistics.median(times[k])
        print(f"{k}: step {ms:.3f} ms median of {args.rounds} rounds x {args.steps} steps "
              f"({' '.join(f'{t:.3f}' for t in times[k])}), {frames / (ms / 1e3):.0f} frames/s")
    med = {k: statistics.median(times[k]) for k in modes}
    print(f"TF32 / IEEE fp32 step time: {med['tf32'] / med['fp32']:.3f}; TF32 / bf16: {med['tf32'] / med['bf16']:.3f}")

    lib = models["tf32"].engine.lib
    print(f"TF32 tensor-core conv launches of one step, median of {args.reps} repetitions:")
    print(f"{'#':>3} {'kernel':<10} {'shape':<36} {'plan':<16} {'us':>8} {'TFLOP/s':>8} {'% of 495':>8}")
    for i, (name, a) in enumerate(calls):
        shape, plan = _describe(lib, name, a)
        tf = flops[i] / us[i] / 1e6
        print(f"{i:>3} {KIND[name]:<10} {shape:<36} {plan:<16} {us[i]:>8.1f} {tf:>8.1f} {100 * tf * 1e12 / TF32_PEAK:>7.1f}%")
    print(f"all {len(calls)} launches: {sum(us) / 1e3:.3f} ms, {sum(flops) / sum(us) / 1e6:.1f} TFLOP/s")

    # every kernel of the step by name: the kernels both modes run are compared; a TF32 kernel slower than its IEEE run
    # is named
    rows = sorted(set(k_fp32) | set(k_tf32), key=lambda n: -(k_fp32.get(n, 0.0) + k_tf32.get(n, 0.0)))
    print(f"device time per step by kernel (torch.profiler, mean of {args.reps} steps):")
    print(f"{'fp32 us':>9} {'tf32 us':>9}  kernel")
    for n in rows:
        print(f"{k_fp32.get(n, 0.0):>9.1f} {k_tf32.get(n, 0.0):>9.1f}  {n[:110]}")
    slower = [n for n in rows if n in k_fp32 and n in k_tf32 and k_tf32[n] > 1.05 * k_fp32[n] + 2.0]
    print("kernels slower in TF32 than in IEEE fp32 (> 5 % and 2 us): " + (", ".join(s[:80] for s in slower) or "none"))
    print(f"sum: fp32 {sum(k_fp32.values()) / 1e3:.3f} ms, tf32 {sum(k_tf32.values()) / 1e3:.3f} ms")


if __name__ == "__main__":
    main()
