"""Times serving independent decoder sessions at the README config (bf16, random weights, cuda_graphs on), one latent
frame per push and session, each session 16 latent frames long, the sessions' starts staggered over the rows:

  batched:    one DecodeStream of B rows; a row whose session ends is restarted (stream.restart) for the next one;
  per-session: B batch_size=1 DecodeStreams pushed in turn; a session that ends is replaced by a new stream, which warms up
              and captures its own graphs again.

For B = 1, 4, 8 and 16 it prints the median device time of one round (one latent frame pushed for every session) over
ROUNDS rounds after WARMUP, and the frames per second delivered over all sessions (the time padding a restarted row
returns is not counted).  Device events, a synchronise after each round; the card's name and power limit are printed with
the numbers.

    python tools/stream_sessions_time.py [--reps 2]
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from magvit2_pytorch_b200 import VideoTokenizer  # noqa: E402
from oracle import weights as W  # noqa: E402
from tests.util import README_LAYERS  # noqa: E402
from tools.stream_time import _card  # noqa: E402

SESSION = 16          # latent frames per session
WARMUP, ROUNDS = 16, 64


def _restarting(B, k):
    """Rows whose session starts at round k > 0: row r at the rounds k = r * SESSION // B (mod SESSION)."""
    return [r for r in range(B) if k > 0 and k % SESSION == r * SESSION // B]


def _round_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _batched(model, codes, B):
    """ms of each round and the frames it delivered: one B-row stream with restarts."""
    tp = model.time_padding
    dec = model.decode_stream(batch_size=B)
    out = []
    for k in range(WARMUP + ROUNDS):
        rows = _restarting(B, k)
        frames = B * model.time_downsample_factor - (B * tp if k == 0 else len(rows) * tp)

        def step():
            if rows:
                dec.restart(rows)
            dec.push(codes[:, k % codes.shape[1]:k % codes.shape[1] + 1])
        out.append((_round_ms(step), frames))
    return out[WARMUP:]


def _per_session(model, codes, B):
    """ms of each round and the frames it delivered: B batch_size=1 streams pushed in turn, a new one per session."""
    tp = model.time_padding
    streams = [model.decode_stream(batch_size=1) for _ in range(B)]
    out = []
    for k in range(WARMUP + ROUNDS):
        rows = _restarting(B, k)
        frames = B * model.time_downsample_factor - (B * tp if k == 0 else len(rows) * tp)

        def step():
            for r in rows:
                streams[r] = model.decode_stream(batch_size=1)
            for r, s in enumerate(streams):
                s.push(codes[r:r + 1, k % codes.shape[1]:k % codes.shape[1] + 1])
        out.append((_round_ms(step), frames))
    return out[WARMUP:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="repetitions of every measurement, alternating the two modes")
    ap.add_argument("--batches", default="1,4,8,16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    torch.manual_seed(0)
    model = VideoTokenizer(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    W.fill_state_dict_(model, 0)
    model = model.cuda().bfloat16().eval()
    model.cuda_graphs = True
    print(f"card: {_card()}")
    print(f"README config, bf16, cuda_graphs on; sessions of {SESSION} latent frames, one per push; "
          f"median over rounds {WARMUP + 1}..{WARMUP + ROUNDS}")
    for B in (int(b) for b in args.batches.split(",")):
        codes = torch.randint(0, 1024, (B, 64, 16, 16), device="cuda")
        res = {"batched": [], "per-session": []}
        for _ in range(args.reps):
            for name, fn in (("batched", _batched), ("per-session", _per_session)):
                rounds = fn(model, codes, B)
                ms = statistics.median(t for t, _ in rounds)
                fps = sum(f for _, f in rounds) / sum(t for t, _ in rounds) * 1e3
                res[name].append((ms, fps))
        for name, rs in res.items():
            ms = ", ".join(f"{m:.2f}" for m, _ in rs)
            fps = ", ".join(f"{f:.0f}" for _, f in rs)
            print(f"  B={B:2d} {name:11s}: {ms} ms per round (median), {fps} frames/s over all sessions", flush=True)


if __name__ == "__main__":
    main()
