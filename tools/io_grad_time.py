"""Times the differentiable entry points at the README config (bf16, random weights, one 17-frame 128 x 128 clip):

  (a) decode forward + backward (latents requiring grad, eval mode), next to the no-grad decode;
  (b) encode forward + backward (video requiring grad, eval mode), next to the no-grad encode;
  (c) the video's data gradient through conv_in alone: the slab kernel's narrow-N launch (TrainRunner.video_dgrad_packed,
      with the transposed weights packed once outside the timed region) against aten.convolution_backward (cuDNN) of the
      same conv, data gradient only.

Device events after a warm-up, median of the repeats; prints the card's name and power limit with the numbers.

    python tools/io_grad_time.py
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
from magvit2_pytorch_b200.train import TrainRunner, transposed_pack  # noqa: E402
from tests.util import README_LAYERS  # noqa: E402

REPEATS = 10


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _ms(fn, repeats=REPEATS):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    torch.manual_seed(0)
    model = VideoTokenizer(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS,
                           use_gan=False, perceptual_loss_weight=0.).cuda().bfloat16().eval()
    video = torch.rand(1, 3, 17, 128, 128, device="cuda")
    with torch.no_grad():
        z = model.encode(video)

    def decode_fb():
        zr = z.detach().requires_grad_(True)
        model.decode(zr).float().square().sum().backward()

    def encode_fb():
        vr = video.detach().requires_grad_(True)
        model.encode(vr).float().square().sum().backward()

    print(f"card: {_card()}")
    with torch.no_grad():
        print(f"decode  no-grad            {_ms(lambda: model.decode(z)):8.2f} ms")
    print(f"decode  forward + backward {_ms(decode_fb):8.2f} ms")
    with torch.no_grad():
        print(f"encode  no-grad            {_ms(lambda: model.encode(video)):8.2f} ms")
    print(f"encode  forward + backward {_ms(encode_fb):8.2f} ms")

    # (c) conv_in's data gradient wrt the video: g (1, 17 + 3, 128, 128, 64) channels-last, time_padding 3 frames dropped
    t_pad = model.time_padding
    w = model.conv_in.conv.weight.detach()
    g = torch.randn(1, 17 + t_pad, 128, 128, 64, device="cuda").bfloat16()
    runner = TrainRunner(model)
    pk = transposed_pack(w, (7, 7, 7), torch.bfloat16)
    x_cf = torch.zeros(1, 3, 17 + t_pad + 6, 128, 128, device="cuda", dtype=torch.bfloat16)     # causal pad materialised
    g_cf = g.permute(0, 4, 1, 2, 3)

    def ours():
        with torch.no_grad():
            return runner.video_dgrad_packed(g, pk, t_pad)

    def aten():
        return torch.ops.aten.convolution_backward(g_cf, x_cf, w, None, [1, 1, 1], [0, 3, 3], [1, 1, 1], False, [0, 0, 0], 1,
                                                   [True, False, False])[0]

    flops = 2.0 * 17 * 128 * 128 * 3 * 64 * 343
    t_ours, t_aten = _ms(ours), _ms(aten)
    print(f"conv_in video dgrad, narrow-N slab launch         {t_ours * 1e3:8.1f} us  ({flops / t_ours / 1e9:6.1f} TFLOP/s)")
    print(f"conv_in video dgrad, aten.convolution_backward    {t_aten * 1e3:8.1f} us  ({flops / t_aten / 1e9:6.1f} TFLOP/s)")
    ref = aten()[:, :, t_pad + 6:].float()
    err = float((ours().float() - ref).abs().max() / ref.abs().max())
    print(f"max |ours - aten| / max |aten| = {err:.2e}")


if __name__ == "__main__":
    main()
