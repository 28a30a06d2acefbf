"""TEST INFRASTRUCTURE ONLY.  tests/golden/mini_gan.pt and mini_gan_bf16.pt: the UNMODIFIED reference
(oracle/ref_loader.py, ``use_gan=True, perceptual_loss_weight=0``) on the `mini` config, with its image discriminator
(M:549-675, 4 blocks, 26.7 M parameters) filled by ``synth_data.fill_discr_``:

* the reference's ``discr.*`` key -> shape map;
* standalone ``discr(images)``: logits, the input gradient of ``logits.sum()`` and parameter-gradient digests, and the
  gradient penalty (M:102-115) of those images with its parameter-gradient digests;
* the seeded train-mode discriminator step (``return_discr_loss``, M:1731-1786) with the penalty off and on: the frame
  indices the reference drew, total / hinge / penalty and the digests of every discriminator gradient;
* the seeded train-mode generator step (``return_loss`` with the adversarial term, M:1826-1896): losses and digests of
  every gradient;
* mini_gan_bf16.pt: the reference's own bf16 run (``model.bfloat16()``) -- standalone logits and the losses of both steps.

Runs only in the build container:   python -m oracle.make_gan_golden
"""
from __future__ import annotations

import os

import torch

import synth_data
from oracle import weights as W
from oracle.make_golden import CONFIGS, GOLDEN_DIR
from oracle.make_train_golden import grad_digest
from oracle.ref_loader import build_reference_tokenizer, load_reference

BASE = "mini"
ISEED = 4321          # standalone discriminator images
STEP_SEED = 7         # torch.manual_seed before each seeded step: the reference's frame choice draws from it


def _record_frames(ref):
    """Wraps the reference's pick_video_frame to record the frame indices it was called with."""
    seen = []
    orig = ref.pick_video_frame

    def pick(video, frame_indices):
        seen.append(frame_indices.clone())
        return orig(video, frame_indices)

    ref.pick_video_frame = pick
    return seen, lambda: setattr(ref, "pick_video_frame", orig)


def _digests(model, prefix=None):
    return {k: (grad_digest(p.grad.detach().float(), 256) if p.grad is not None else None)
            for k, p in model.named_parameters() if prefix is None or k.startswith(prefix)}


def _zero(model):
    for _, p in model.named_parameters():          # the reference's parameters() lists the generator only (M:1460)
        p.grad = None


def _images(dtype=torch.float32):
    g = torch.Generator(device="cpu")
    g.manual_seed(ISEED)
    return torch.randn(2, 3, 32, 32, generator=g).to(dtype)


def _build(cfg, kwargs):
    torch.manual_seed(0)
    model = build_reference_tokenizer(**kwargs)
    W.fill_state_dict_(model, cfg["wseed"])
    synth_data.fill_discr_(model, cfg["wseed"])
    return model


def _steps(model, video, ref, penalty_on=True, digests=True):
    out = {}
    seen, restore = _record_frames(ref)
    try:
        model.train()
        for gp in ((False, True) if penalty_on else (False,)):
            _zero(model)
            torch.manual_seed(STEP_SEED)
            total, bd = model(video, return_discr_loss=True, apply_gradient_penalty=gp)
            ent = dict(frames=seen[-2:][0].clone(), total=total.detach().float().clone(), hinge=bd.discr_loss.detach().float().clone(),
                       penalty=torch.as_tensor(bd.gradient_penalty).detach().float().clone())
            if digests:
                total.backward()
                ent["grads"] = _digests(model, "discr.")
            out["discr_gp" if gp else "discr"] = ent
        _zero(model)
        torch.manual_seed(STEP_SEED)
        total, bd = model(video, return_loss=True)
        ent = dict(frames=seen[-1].clone(), total=total.detach().float().clone(), recon=bd.recon_loss.detach().float().clone(),
                   aux=torch.as_tensor(bd.lfq_aux_loss).detach().float().clone(),
                   gen=bd.adversarial_gen_loss.detach().float().clone())
        if digests:
            total.backward()
            ent["grads"] = _digests(model)
        out["gen"] = ent
    finally:
        restore()
    return out


def make():
    cfg = CONFIGS[BASE]
    kwargs = dict(cfg["kwargs"], use_gan=True, perceptual_loss_weight=0.)
    ref = load_reference()
    model = _build(cfg, kwargs)
    video = W.synth_video(*cfg["video"][:3], cfg["video"][3], seed=cfg["vseed"])
    out = dict(name="mini_gan", kwargs=kwargs, video_shape=tuple(cfg["video"]), wseed=cfg["wseed"], vseed=cfg["vseed"],
               iseed=ISEED, step_seed=STEP_SEED)
    out["discr_shapes"] = {k: tuple(v.shape) for k, v in model.state_dict().items() if k.startswith("discr.")}
    d = model.discr

    imgs = _images().requires_grad_(True)
    _zero(model)
    logits = d(imgs)
    logits.sum().backward()
    out["standalone"] = dict(logits=logits.detach().clone(), grad_images=grad_digest(imgs.grad.detach(), 256),
                             grads=_digests(d))
    _zero(model)
    x = _images().requires_grad_(True)
    gp = ref.gradient_penalty(x, d(x))
    gp.backward()
    out["penalty"] = dict(value=gp.detach().clone(), grads=_digests(d))
    out.update(_steps(model, video, ref))
    out["reference_commit"] = "a00519fa (v0.5.1)"
    out["third_party"] = "oracle/shims (restated LFQ/TaylorSeriesLinearAttn; real packages unavailable)"
    path = os.path.join(GOLDEN_DIR, "mini_gan.pt")
    torch.save(out, path)
    print(f"[golden] mini_gan: logits {out['standalone']['logits'].tolist()} penalty {out['penalty']['value'].item():.6f}; "
          f"discr {out['discr']['total'].item():.6f} (gp {out['discr_gp']['penalty'].item():.6f}); gen total "
          f"{out['gen']['total'].item():.6f} gen {out['gen']['gen'].item():.6f}; frames {out['gen']['frames'].tolist()}; "
          f"{sum(p.numel() for p in d.parameters()) / 1e6:.1f} M discr params; {os.path.getsize(path) / 1e3:.0f} KB")

    model16 = _build(cfg, kwargs).bfloat16()
    with torch.no_grad():
        logits16 = model16.discr(_images(torch.bfloat16)).float()
    out16 = dict(name="mini_gan_bf16", kwargs=kwargs, logits=logits16.clone())
    out16.update(_steps(model16, video.bfloat16(), ref, penalty_on=False, digests=False))
    path = os.path.join(GOLDEN_DIR, "mini_gan_bf16.pt")
    torch.save(out16, path)
    print(f"[golden] mini_gan_bf16: logits {logits16.tolist()}; discr {out16['discr']['total'].item():.6f}; gen total "
          f"{out16['gen']['total'].item():.6f}; {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    make()
