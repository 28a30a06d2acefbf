"""Times the perceptual-loss pieces at the README config (4 clips x 17 frames x 128^2, bf16, a full-width VGG16 layout with
the reference's truncated classifier, synth_data.build_vgg): the VGG forward on 8 frames, the VGG data gradient on 4
frames, one last-layer weight gradient of the adaptive weight (two per step), the generator step with and without the
perceptual and adaptive terms, and the VGG convs' rate from shape-derived FLOPs.

Device events after a warm-up; prints the card's name and power limit with the numbers.

    python tools/perceptual_step_time.py [--clips 4] [--iters 5]
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth_data  # noqa: E402
from magvit2_pytorch_b200 import VideoTokenizer  # noqa: E402
from magvit2_pytorch_b200 import vgg as V  # noqa: E402
from tools.gan_step_time import README_LAYERS, _card, _time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=4)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: timings are only taken on the GPU")
    torch.manual_seed(0)
    vgg = synth_data.fill_vgg_(synth_data.build_vgg(synth_data.VGG16_CFG, 4096))
    kw = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
    m = VideoTokenizer(**kw, vgg=vgg)
    synth_data.fill_state_dict_(m)
    synth_data.fill_discr_(m)
    m = m.cuda().bfloat16().train()
    m.vgg.eval()                                   # dropout off: the timed steps do the same work each time
    video = synth_data.synth_video(args.clips, 3, 17, 128).cuda().bfloat16()
    frames8 = video[:, :, :2].transpose(1, 2).reshape(-1, 3, 128, 128).contiguous()[:8]
    frames4 = frames8[:4].contiguous()
    cache = m._vgg_cache

    def vgg_fwd():
        V.VggRunner(m.vgg, (128, 128), 3, cache).forward(frames8, record=False)

    runners = []

    def vgg_bwd_prep():
        r = V.VggRunner(m.vgg, (128, 128), 3, cache)
        f = r.forward(frames4)
        runners.append((r, torch.ones_like(f)))

    def vgg_bwd():
        r, g = runners.pop()
        r.backward(g)

    def zero():
        for _, p in m.named_parameters():
            p.grad = None

    def gen_step(vgg_on):
        zero()
        # without: the step of a perceptual_loss_weight=0 GAN model (adaptive weight 1)
        m.use_vgg, m.perceptual_loss_weight = vgg_on, 0.1 if vgg_on else 0.
        try:
            loss, _ = m(video, return_loss=True)
        finally:
            m.use_vgg, m.perceptual_loss_weight = True, 0.1
        loss.backward()

    with torch.no_grad():
        t_fwd = _time(vgg_fwd, args.iters * 4)
        for _ in range(args.iters * 4 + 2):
            vgg_bwd_prep()
        t_bwd = _time(vgg_bwd, args.iters * 4)
        # FLOPs of the VGG's convs per forward on 8 frames, from the shapes (every wgmma launch: 3x3 convs and the Linears)
        eng = cache.engine
        eng._prof = []
        vgg_fwd()
        torch.cuda.synchronize()
        recs, eng._prof = eng._prof, None
    # the adaptive weight's two last-layer gradients (TrainRunner.last_layer_weight_grad), on one saved training forward
    from magvit2_pytorch_b200.train import TrainRunner, train_forward
    runner = TrainRunner(m)
    recon, _, _, _ = train_forward(m, video, runner=runner)
    g_recon = torch.randn_like(recon)
    with torch.no_grad():
        t_last = _time(lambda: runner.last_layer_weight_grad(g_recon), args.iters * 4)
    del runner, recon
    conv_ms = sum(e0.elapsed_time(e1) for e0, e1, *_ in recs)
    conv_flops = sum(r[2] for r in recs)
    res = dict(card=_card(), clips=args.clips, vgg_params_M=round(sum(p.numel() for p in vgg.parameters()) / 1e6, 1),
               vgg_forward_8_frames_ms=round(t_fwd, 3), vgg_data_grad_4_frames_ms=round(t_bwd, 3),
               vgg_wgmma_convs_8_frames=dict(launches=len(recs), gflop=round(conv_flops / 1e9, 1), ms=round(conv_ms, 3),
                                             tflops=round(conv_flops / conv_ms / 1e9, 1) if conv_ms else None),
               last_layer_weight_grad_ms=round(t_last, 2),
               gen_step_ms=round(_time(lambda: gen_step(True), args.iters), 1),
               gen_step_no_perceptual_ms=round(_time(lambda: gen_step(False), args.iters), 1))
    print(res)


if __name__ == "__main__":
    main()
