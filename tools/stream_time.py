"""Times streaming decode and tokenize at the README config (bf16, random weights) for B = 1 and 4:

  (a) pushing one latent frame to a DecodeStream at prefix lengths 1..16, next to decode_from_code_indices of the whole
      prefix (what a frame-by-frame consumer without streams has to call);
  (b) a 1 + 4 * 63-frame video through a TokenizeStream (1 frame, then 4 per push): frames/s and the peak allocation, next
      to one tokenize of the same video.

Device events after a warm-up; prints the card's name and power limit with the numbers.

    python tools/stream_time.py
"""
from __future__ import annotations

import os
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
        for _ in range(2):                                   # warm-up: every shape below once
            dec = model.decode_stream(batch_size=B)
            for k in range(16):
                dec.push(codes[:, k:k + 1])
                model.decode_from_code_indices(codes[:, :k + 1])
        torch.cuda.synchronize()
        print(f"(a) B={B}: ms per step, one latent frame pushed vs decode_from_code_indices of the prefix")
        dec = model.decode_stream(batch_size=B)
        for k in range(16):
            t_push, _ = _ms(lambda: dec.push(codes[:, k:k + 1]))
            t_full, _ = _ms(lambda: model.decode_from_code_indices(codes[:, :k + 1]))
            print(f"  prefix {k + 1:2d}: push {t_push:8.2f}  whole prefix {t_full:8.2f}")
        video = W.synth_video(B, 3, 1 + 4 * 63, 128, seed=1).cuda().bfloat16()

        def stream():
            enc = model.tokenize_stream(batch_size=B)
            out = [enc.push(video[:, :, :1])]
            for t in range(1, video.shape[2], 4):
                out.append(enc.push(video[:, :, t:t + 4]))
            return torch.cat(out, 1)

        for name, fn in (("stream", stream), ("one-shot", lambda: model.tokenize(video))):
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            ms, _ = _ms(fn)
            peak = torch.cuda.max_memory_allocated() - base
            print(f"(b) B={B} tokenize {name:8s}: {B * video.shape[2] / ms * 1e3:9.1f} frames/s, peak +{peak / 2**20:8.1f} MiB")


if __name__ == "__main__":
    main()
