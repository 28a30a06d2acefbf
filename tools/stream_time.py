"""Times streaming decode and tokenize at the README config (bf16, random weights) for B = 1 and 4, each push with
cuda_graphs off (eager) and on (replayed push plans, stream.PushPlan):

  (a) pushing one latent frame to a DecodeStream at prefix lengths 1..16, next to decode_from_code_indices of the whole
      prefix (what a frame-by-frame consumer without streams has to call).  With graphs the first pushes run eagerly
      while the stream's histories fill, the next one warms up, the one after is captured ("capture"), the rest replay;
  (b) a 1 + 4 * 63-frame video through a TokenizeStream (1 frame, then 4 per push): the median time of the 4-frame pushes
      from the 8th on, and frames/s and the peak allocation of the whole stream, warm-up and capture included, next to one
      tokenize of the same video.

Device events, a synchronise after each timed call; prints the card's name and power limit with the numbers.

    python tools/stream_time.py
"""
from __future__ import annotations

import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from magvit2_pytorch_b200 import VideoTokenizer  # noqa: E402
from oracle import weights as W  # noqa: E402
from tests.util import README_LAYERS  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def _decode_pushes(model, codes, graphs):
    """ms of each one-frame push of a new DecodeStream, and whether it was captured."""
    model.cuda_graphs = graphs
    dec = model.decode_stream(batch_size=codes.shape[0])
    out = []
    for k in range(codes.shape[1]):
        n0 = dec.captures
        t, _ = _ms(lambda: dec.push(codes[:, k:k + 1]))
        out.append((t, dec.captures > n0))
    model.cuda_graphs = False
    return out


def _tokenize_stream(model, video, graphs, times=None):
    """Codes of `video` through a new TokenizeStream: 1 frame, then 4 per push; `times` gets each push's ms."""
    model.cuda_graphs = graphs
    enc = model.tokenize_stream(batch_size=video.shape[0])
    out = []
    for t in [0] + list(range(1, video.shape[2], 4)):
        chunk = video[:, :, t:t + (1 if t == 0 else 4)]
        if times is None:
            out.append(enc.push(chunk))
        else:
            ms, c = _ms(lambda: enc.push(chunk))
            times.append(ms)
            out.append(c)
    model.cuda_graphs = False
    return torch.cat(out, 1)


def main():
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    torch.manual_seed(0)
    model = VideoTokenizer(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    W.fill_state_dict_(model, 0)
    model = model.cuda().bfloat16().eval()
    print(f"card: {_card()}")
    for B in (1, 4):
        codes = torch.randint(0, 1024, (B, 16, 16, 16), device="cuda")
        for graphs in (False, True):                         # warm-up: every shape below once
            _decode_pushes(model, codes, graphs)
        for k in range(16):
            model.decode_from_code_indices(codes[:, :k + 1])
        torch.cuda.synchronize()
        print(f"(a) B={B}: ms per step, one latent frame pushed (graphs off / on) vs decode_from_code_indices of the prefix")
        off, on = _decode_pushes(model, codes, False), _decode_pushes(model, codes, True)
        for k in range(16):
            t_full, _ = _ms(lambda: model.decode_from_code_indices(codes[:, :k + 1]))
            tag = " (capture)" if on[k][1] else ""
            print(f"  prefix {k + 1:2d}: push {off[k][0]:8.2f} / {on[k][0]:8.2f}  whole prefix {t_full:8.2f}{tag}")
        video = W.synth_video(B, 3, 1 + 4 * 63, 128, seed=1).cuda().bfloat16()
        for graphs in (False, True):
            times = []
            _tokenize_stream(model, video, graphs, times)
            print(f"(b) B={B} tokenize push of 4 frames, graphs {'on ' if graphs else 'off'}: median "
                  f"{statistics.median(times[8:]):7.2f} ms over pushes 9..64")
        runs = (("stream, graphs off", lambda: _tokenize_stream(model, video, False)),
                ("stream, graphs on", lambda: _tokenize_stream(model, video, True)),
                ("one-shot", lambda: model.tokenize(video)))
        for name, fn in runs:
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            ms, _ = _ms(fn)
            peak = torch.cuda.max_memory_allocated() - base
            print(f"(b) B={B} tokenize {name:18s}: {B * video.shape[2] / ms * 1e3:9.1f} frames/s, "
                  f"peak +{peak / 2**20:8.1f} MiB")


if __name__ == "__main__":
    main()
