"""bf16 against fp16 on the benchmark's step: README config, 4 clips of 3x17x128x128 (the benchmark's weight and input
seeds), tokenize + decode_from_code_indices through StreamLanes(tok, 3) with CUDA graphs on, as bench.py times it.  Both
models live in one process and are timed in alternating rounds (--rounds each, --steps steps per round after a warm-up
that captures every lane's graphs), so drift of the shared card's clocks hits both alike.  Then the per-launch times of
the tensor-core convs of one step of each dtype, the way tools/slab_conv_time.py takes them (device events around every
launch, each repetition queued behind a GPU spin), side by side, and the device time of every kernel of the step by name
(torch.profiler), so that a difference between the dtypes can be traced to its kernels.  The card's name, power limit
and the median SM clock during the timed rounds are printed with the numbers.

    python tools/f16_time.py [--rounds 5] [--steps 100] [--reps 30]
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth_data as Wt  # noqa: E402
from bench import README_KW, ClockSampler  # noqa: E402
from magvit2_pytorch_b200 import StreamLanes, VideoTokenizer  # noqa: E402
from tools.slab_conv_time import KIND, _card, _describe, _RecordingLib  # noqa: E402

CLIPS, FRAMES = 4, 17


def _model(dtype):
    torch.manual_seed(0)
    m = VideoTokenizer(**README_KW)
    Wt.fill_state_dict_(m, 0)
    m = m.cuda().to(dtype).eval()
    m.cuda_graphs = True
    return m


def _step(model):
    def step(v):
        codes = model.tokenize(v)
        return codes, model.decode_from_code_indices(codes)
    return step


def _round(lanes, step, batches, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(steps):
        lanes.run(step, batches[i % len(batches)])
    lanes.join()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _per_launch(model, video, reps):
    """[(name, args)] of one step's tensor-core conv launches and their median microseconds over `reps` repetitions"""
    eng = model.engine
    step = _step(model)
    model.cuda_graphs = False                        # eager calls: the events bracket each launch
    for _ in range(2):
        step(video)
    torch.cuda.synchronize()
    rec = _RecordingLib(eng.lib)
    eng.lib = rec
    eng._prof = []
    try:
        step(video)
        torch.cuda.synchronize()
        calls = list(rec.calls)
        eng._prof = []
        for _ in range(reps):
            torch.cuda._sleep(int(100e6))
            step(video)
        torch.cuda.synchronize()
        prof = eng._prof
    finally:
        eng._prof = None
        eng.lib = rec._lib
        model.cuda_graphs = True
    n = len(calls)
    assert n and len(prof) == n * reps, (n, len(prof))
    us = [statistics.median(prof[r * n + i][0].elapsed_time(prof[r * n + i][1]) * 1e3 for r in range(reps)) for i in range(n)]
    return calls, us, [prof[i][2] for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating timed rounds per dtype (>= 3)")
    ap.add_argument("--steps", type=int, default=100, help="steps per round")
    ap.add_argument("--reps", type=int, default=30, help="repetitions of the per-launch conv timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert args.rounds >= 3

    models = {"bf16": _model(torch.bfloat16), "fp16": _model(torch.float16)}
    batches = {k: [Wt.synth_video(CLIPS, 3, FRAMES, 128, seed=1000 + i).cuda().to(m.dtype) for i in range(2)]
               for k, m in models.items()}
    lanes = {k: StreamLanes(m, 3) for k, m in models.items()}
    steps = {k: _step(m) for k, m in models.items()}
    with torch.no_grad():
        for k in models:
            for i in range(9):                        # every lane: plain call, graph capture, first replay
                lanes[k].run(steps[k], batches[k][i % 2])
            lanes[k].join()
        torch.cuda.synchronize()
        clk = ClockSampler(torch.cuda.current_device())
        clk.start()
        clk.begin()
        times = {k: [] for k in models}
        try:
            for _ in range(args.rounds):
                for k in models:
                    times[k].append(_round(lanes[k], steps[k], batches[k], args.steps))
        finally:
            clocks = clk.stop()
        per = {k: _per_launch(m, batches[k][0], args.reps) for k, m in models.items()}

    print(f"card: {_card()}  (name, power limit, max SM clock)")
    print(f"SM clock during the timed rounds: median {clocks.get('sm_mhz')} MHz of {clocks.get('sm_max_mhz')} "
          f"({clocks.get('samples')} samples, reasons {clocks.get('reasons')})")
    frames = CLIPS * FRAMES
    for k in models:
        ms = statistics.median(times[k])
        print(f"{k}: step {ms:.3f} ms median of {args.rounds} rounds x {args.steps} steps "
              f"({' '.join(f'{t:.3f}' for t in times[k])}), {frames / (ms / 1e3):.0f} frames/s")
    ratio = statistics.median(times["fp16"]) / statistics.median(times["bf16"])
    print(f"fp16 / bf16 step time: {ratio:.3f}")

    (cb, ub, fb), (cf, uf, _) = per["bf16"], per["fp16"]
    assert [(n, _describe(models['bf16'].engine.lib, n, a)[0]) for n, a in cb] == \
        [(n, _describe(models['fp16'].engine.lib, n, a)[0]) for n, a in cf], "the two dtypes launch different convs"
    lib = models["bf16"].engine.lib
    print(f"per launch, median of {args.reps} repetitions:")
    print(f"{'#':>3} {'kernel':<10} {'shape':<36} {'plan':<16} {'bf16 us':>8} {'fp16 us':>8} {'ratio':>6} {'fp16 TFLOP/s':>12}")
    for i, (name, a) in enumerate(cb):
        shape, plan = _describe(lib, name, a)
        print(f"{i:>3} {KIND[name]:<10} {shape:<36} {plan:<16} {ub[i]:>8.1f} {uf[i]:>8.1f} {uf[i] / ub[i]:>6.3f} "
              f"{fb[i] / uf[i] / 1e6:>12.1f}")
    print(f"all {len(cb)} launches: bf16 {sum(ub) / 1e3:.3f} ms, fp16 {sum(uf) / 1e3:.3f} ms, ratio {sum(uf) / sum(ub):.3f}")

    # every kernel of the step, tensor-core convs and CUDA-core ops alike: device time per kernel name (torch.profiler, in
    # a pass of its own), the fp16 kernels matched to their bf16 twins by name
    prof = {k: _kernel_times(m, batches[k][0], args.reps) for k, m in models.items()}
    rows = []
    for name, us_b in prof["bf16"].items():
        twin = _f16_name(name)
        us_f = prof["fp16"].pop(twin, None)
        rows.append((name, us_b, us_f))
    rows += [(f"(fp16 only) {n}", None, u) for n, u in prof["fp16"].items()]
    rows.sort(key=lambda r: -abs((r[2] or 0.0) - (r[1] or 0.0)))
    print(f"device time per step by kernel (torch.profiler, mean of {args.reps} steps), largest fp16 - bf16 difference first:")
    print(f"{'bf16 us':>9} {'fp16 us':>9} {'diff us':>8}  kernel")
    for name, ub_, uf_ in rows:
        print(f"{ub_ or 0:>9.1f} {uf_ or 0:>9.1f} {(uf_ or 0) - (ub_ or 0):>8.1f}  {name[:110]}")
    print(f"sum: bf16 {sum(r[1] or 0 for r in rows) / 1e3:.3f} ms, fp16 {sum(r[2] or 0 for r in rows) / 1e3:.3f} ms")


def _f16_name(name):
    """the name of the fp16 twin of a bf16 kernel"""
    for k in ("tc_slab_kernel", "tc_conv_kernel", "attention_mma_kernel", "attention_small_kernel"):
        if k + "<" in name:
            return name.replace(k, k[:-len("kernel")] + "f16_kernel", 1)
    return name.replace("__nv_bfloat16", "__half")


def _kernel_times(model, video, reps):
    """{kernel name: mean device microseconds per step} of eager tokenize + decode"""
    from torch.profiler import ProfilerActivity, profile
    step = _step(model)
    model.cuda_graphs = False
    step(video)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            step(video)
        torch.cuda.synchronize()
    model.cuda_graphs = True
    out = {}
    for e in p.key_averages():
        if e.device_type.name == "CUDA" and e.self_device_time_total > 0:
            out[e.key] = out.get(e.key, 0.0) + e.self_device_time_total / reps
    return out


if __name__ == "__main__":
    main()
