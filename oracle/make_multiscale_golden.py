"""TEST INFRASTRUCTURE ONLY.  tests/golden/mini_ms_gan.pt, mini_ms_gan_vgg.pt and mini_ms_vgg.pt: the UNMODIFIED reference
(oracle/ref_loader.py) on the `mini` config with two multiscale discriminators (``multiscale_discrs=``, M:1085,
M:1429-1441; oracle/video_discr.py) and ``multiscale_adversarial_loss_weight=0.5``, in three variants:

* ms_gan: the image GAN without a perceptual term (multiscale adaptive weights 1.);
* ms_gan_vgg: the image GAN and a VGG module (synth_data.build_vgg, the narrow layout of make_vgg_golden.py);
* ms_vgg: a VGG without the image GAN (``adversarial_loss_weight=0``): the multiscale generator terms take the perceptual
  term's frame pick, and the reference's discriminator step refuses the model (``assert self.has_gan``, M:1732).

Each records, in fp32: the seeded train-mode generator step (``return_loss``, M:1788-1896; the VGG in eval(), dropout off):
the frame indices of the perceptual and image-GAN picks, every LossBreakdown field including both multiscale lists, and the
digests of every parameter's gradient (the VGG's excepted; the multiscale discriminators get none: the reference's generator
loop never calls them, M:1852-1853); the eval-mode losses; the seeded discriminator step (``return_discr_loss`` with the
gradient penalty, M:1731-1786): total, DiscrLossBreakdown and the digests of every discriminator gradient.  Under "bf16": the
reference's own bf16 run (``model.bfloat16()``) of the generator step and, without the penalty, the discriminator step.

Runs only in the build container:   python -m oracle.make_multiscale_golden
"""
from __future__ import annotations

import os

import torch

import synth_data
from oracle import weights as W
from oracle.make_gan_golden import STEP_SEED, _digests, _record_frames, _zero
from oracle.make_golden import CONFIGS, GOLDEN_DIR
from oracle.make_vgg_golden import VARIANTS as VGG_VARIANTS, VSEED, make_vgg
from oracle.ref_loader import build_reference_tokenizer, load_reference
from oracle.video_discr import SPECS, make_video_discrs

BASE = "mini"
MSEED = 5             # oracle.video_discr.make_video_discrs seed
MS_WEIGHT = 0.5       # multiscale_adversarial_loss_weight: not 1, so that the goldens pin where it is applied
VARIANTS = {
    "mini_ms_gan": dict(vgg=None, kwargs=dict(use_gan=True, perceptual_loss_weight=0.)),
    "mini_ms_gan_vgg": dict(vgg="mini_vgg_narrow", kwargs=dict(use_gan=True, perceptual_loss_weight=0.1)),
    "mini_ms_vgg": dict(vgg="mini_vgg_narrow", kwargs=dict(use_gan=True, perceptual_loss_weight=0.1, adversarial_loss_weight=0.)),
}


def _f(x):
    return torch.as_tensor(x).detach().float().clone()


def _build(cfg, kwargs, spec):
    torch.manual_seed(0)
    vgg = make_vgg(VGG_VARIANTS[spec["vgg"]]) if spec["vgg"] else None
    model = build_reference_tokenizer(**kwargs, vgg=vgg, multiscale_discrs=tuple(make_video_discrs(3, MSEED)))
    W.fill_state_dict_(model, cfg["wseed"])
    synth_data.fill_discr_(model, cfg["wseed"])
    assert model.has_multiscale_discrs and len(model.multiscale_discrs) == len(SPECS)
    return model


def _gen_step(model, video, ref, digests=True):
    seen, restore = _record_frames(ref)
    try:
        model.train()
        if model.use_vgg:
            model.vgg.eval()
        _zero(model)
        torch.manual_seed(STEP_SEED)
        total, bd = model(video, return_loss=True)
        ent = dict(frames=[s.clone() for s in seen], total=_f(total), recon=_f(bd.recon_loss), aux=_f(bd.lfq_aux_loss),
                   perceptual=_f(bd.perceptual_loss), gen=_f(bd.adversarial_gen_loss), adaptive=_f(bd.adaptive_adversarial_weight),
                   ms_gen=torch.stack([_f(x) for x in bd.multiscale_gen_losses]),
                   ms_weights=torch.stack([_f(x) for x in bd.multiscale_gen_adaptive_weights]))
        if model.use_vgg:
            ent["perceptual_frames"] = seen[0].clone()        # M:1792: input and recon frames, one draw
        if model.has_gan:
            ent["gen_frames"] = seen[-1].clone()              # M:1827
        if digests:
            total.backward()
            ent["grads"] = {k: v for k, v in _digests(model).items() if not k.startswith("vgg.")}
        model.eval()
        torch.manual_seed(STEP_SEED)
        with torch.no_grad():
            total, bd = model(video, return_loss=True)
        ent["eval"] = dict(total=_f(total), perceptual=_f(bd.perceptual_loss), gen=_f(bd.adversarial_gen_loss),
                           ms_gen=torch.stack([_f(x) for x in bd.multiscale_gen_losses]),
                           ms_weights=torch.tensor([float(x) for x in bd.multiscale_gen_adaptive_weights]))
    finally:
        restore()
    return ent


def _discr_step(model, video, ref, gp, digests=True):
    seen, restore = _record_frames(ref)
    try:
        model.train()
        _zero(model)
        torch.manual_seed(STEP_SEED)
        total, bd = model(video, return_discr_loss=True, apply_gradient_penalty=gp)
        ent = dict(frames=seen[0].clone(), total=_f(total), hinge=_f(bd.discr_loss), penalty=_f(bd.gradient_penalty),
                   ms_discr=torch.stack([_f(x) for x in bd.multiscale_discr_losses]))
        if digests:
            total.backward()
            ent["grads"] = {k: v for k, v in _digests(model).items() if k.startswith(("discr.", "multiscale_discrs."))}
    finally:
        restore()
    return ent


def make(name):
    spec = VARIANTS[name]
    cfg = CONFIGS[BASE]
    kwargs = dict(cfg["kwargs"], multiscale_adversarial_loss_weight=MS_WEIGHT, **spec["kwargs"])
    ref = load_reference()
    video = W.synth_video(*cfg["video"][:3], cfg["video"][3], seed=cfg["vseed"])
    out = dict(name=name, kwargs=kwargs, mseed=MSEED, video_shape=tuple(cfg["video"]), wseed=cfg["wseed"], vseed=cfg["vseed"],
               step_seed=STEP_SEED)
    if spec["vgg"]:
        out.update(vgg=dict(VGG_VARIANTS[spec["vgg"]]), vseed_vgg=VSEED)
    model = _build(cfg, kwargs, spec)
    out["ms_shapes"] = {k: tuple(v.shape) for k, v in model.state_dict().items() if k.startswith("multiscale_discrs.")}
    out["gen"] = _gen_step(model, video, ref)
    if model.has_gan:
        out["discr"] = _discr_step(model, video, ref, gp=True)

    model16 = _build(cfg, kwargs, spec).bfloat16()
    out["bf16"] = dict(gen=_gen_step(model16, video.bfloat16(), ref, digests=False))
    if model16.has_gan:
        out["bf16"]["discr"] = _discr_step(model16, video.bfloat16(), ref, gp=False, digests=False)
    out["reference_commit"] = "a00519fa (v0.5.1)"
    out["third_party"] = "oracle/shims (restated LFQ/TaylorSeriesLinearAttn; real packages unavailable)"
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    torch.save(out, path)
    g = out["gen"]
    d = f"; discr total {out['discr']['total'].item():.6f} ms {out['discr']['ms_discr'].tolist()}" if "discr" in out else ""
    print(f"[golden] {name}: total {g['total'].item():.6f} perceptual {g['perceptual'].item():.6f} gen {g['gen'].item():.6f} "
          f"adaptive {g['adaptive'].item():.6f} ms_gen {g['ms_gen'].tolist()} ms_weights {g['ms_weights'].tolist()}{d}; "
          f"bf16 total {out['bf16']['gen']['total'].item():.6f}; {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    for n in VARIANTS:
        make(n)
