"""Times the GAN training pieces at the README config (4 clips x 17 frames x 128^2, bf16, discriminator dim 512):
the discriminator forward on 4 frames, the generator step with and without the adversarial term, the discriminator step
with and without the gradient penalty, and the discriminator convs' rate from shape-derived FLOPs.

Device events after a warm-up; prints the card's name and power limit with the numbers.  Penalty steps run the torch
restatement under double backward (library code, no speed claim).

    python tools/gan_step_time.py [--clips 4] [--iters 5]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth_data  # noqa: E402
from magvit2_pytorch_b200 import VideoTokenizer  # noqa: E402

README_LAYERS = (
    "residual", "compress_space", ("consecutive_residual", 2), "compress_space",
    ("consecutive_residual", 2), "linear_attend_space", "compress_space",
    ("consecutive_residual", 2), "attend_space", "compress_time",
    ("consecutive_residual", 2), "compress_time", ("consecutive_residual", 2), "attend_time",
)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=4)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: timings are only taken on the GPU")
    torch.manual_seed(0)
    kw = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS, perceptual_loss_weight=0.)
    m = VideoTokenizer(**kw)
    synth_data.fill_state_dict_(m)
    synth_data.fill_discr_(m)
    m = m.cuda().bfloat16().train()
    video = synth_data.synth_video(args.clips, 3, 17, 128).cuda().bfloat16()
    frames = video[:, :, 0].contiguous()
    d = m.discr

    def zero():
        for _, p in m.named_parameters():
            p.grad = None

    def gen_step(adv):
        zero()
        m.has_gan = adv               # without: the step of a use_gan=False model (no discriminator call)
        try:
            loss, _ = m(video, return_loss=True)
        finally:
            m.has_gan = True
        loss.backward()

    def discr_step(gp):
        zero()
        loss, _ = m(video, return_discr_loss=True, apply_gradient_penalty=gp)
        loss.backward()

    with torch.no_grad():
        t_fwd = _time(lambda: d(frames), args.iters * 4)
    # FLOPs of the discriminator's convs (3x3, 1x1 / 2x2 stride 2, to_logits) per forward, from the shapes
    eng = d._pack_cache.engine
    eng._prof = []
    with torch.no_grad():
        d(frames)
    torch.cuda.synchronize()
    recs, eng._prof = eng._prof, None
    conv_ms = sum(e0.elapsed_time(e1) for e0, e1, *_ in recs)
    conv_flops = sum(r[2] for r in recs)
    res = dict(card=_card(), clips=args.clips, discr_params_M=round(sum(p.numel() for p in d.parameters()) / 1e6, 1),
               discr_forward_ms=round(t_fwd, 3),
               discr_wgmma_convs=dict(launches=len(recs), gflop=round(conv_flops / 1e9, 1), ms=round(conv_ms, 3),
                                      tflops=round(conv_flops / conv_ms / 1e9, 1) if conv_ms else None),
               gen_step_ms=round(_time(lambda: gen_step(True), args.iters), 1),
               gen_step_no_adversarial_ms=round(_time(lambda: gen_step(False), args.iters), 1),
               discr_step_ms=round(_time(lambda: discr_step(False), args.iters), 1),
               discr_step_penalty_ms=round(_time(lambda: discr_step(True), args.iters), 1))
    print(res)


if __name__ == "__main__":
    main()
