"""TEST INFRASTRUCTURE ONLY.  tests/golden/mini_vgg16.pt and mini_vgg_narrow.pt: the UNMODIFIED reference
(oracle/ref_loader.py, ``use_gan=True, perceptual_loss_weight=0.1, vgg=<module>``, M:1081, M:1397-1405) on the `mini`
config, with its discriminator filled by ``synth_data.fill_discr_`` and a VGG built by ``synth_data.build_vgg`` and filled
by ``synth_data.fill_vgg_``:

* vgg16: torchvision's VGG16 layout with the classifier truncated as at M:1403 -- a 1x1 last feature map at 32 px, so the
  adaptive average pool replicates it 49 times;
* narrow: a narrow VGG with three pools and the full classifier -- a 4x4 last feature map pooled to 7x7, like the 128-px
  case of VGG16.

Each records, in fp32: the standalone features of seeded images and the input-gradient digest of ``features.sum()``; the
seeded train-mode generator step (``return_loss``, M:1788-1896) with the VGG in eval() (dropout off): the frame indices of
the perceptual and adversarial terms, total / recon / aux / perceptual / gen losses, the adaptive weight and the digests of
every generator and discriminator gradient (the VGG's are not recorded: the device path gives it none); the eval-mode
losses.  Under "bf16": the reference's own bf16 run (``model.bfloat16()``) -- standalone features and the step's losses.

Runs only in the build container:   python -m oracle.make_vgg_golden
"""
from __future__ import annotations

import os

import torch

import synth_data
from oracle import weights as W
from oracle.make_gan_golden import ISEED, STEP_SEED, _record_frames
from oracle.make_golden import CONFIGS, GOLDEN_DIR
from oracle.make_train_golden import grad_digest
from oracle.ref_loader import build_reference_tokenizer, load_reference

BASE = "mini"
VSEED = 11            # synth_data.fill_vgg_ seed
VARIANTS = {
    "mini_vgg16": dict(cfg=synth_data.VGG16_CFG, hidden=4096, num_classes=None),
    "mini_vgg_narrow": dict(cfg=(16, "M", 32, "M", 64, 64, "M"), hidden=64, num_classes=32),
}


def make_vgg(spec):
    torch.manual_seed(0)
    return synth_data.fill_vgg_(synth_data.build_vgg(spec["cfg"], spec["hidden"], spec["num_classes"]), VSEED)


def _images(dtype=torch.float32):
    g = torch.Generator(device="cpu")
    g.manual_seed(ISEED)
    return torch.randn(2, 3, 32, 32, generator=g).to(dtype)


def _build(cfg, kwargs, spec):
    torch.manual_seed(0)
    model = build_reference_tokenizer(**kwargs, vgg=make_vgg(spec))
    W.fill_state_dict_(model, cfg["wseed"])
    synth_data.fill_discr_(model, cfg["wseed"])
    return model


def _gen_step(model, video, ref, digests=True):
    seen, restore = _record_frames(ref)
    try:
        model.train()
        model.vgg.eval()
        for _, p in model.named_parameters():
            p.grad = None
        torch.manual_seed(STEP_SEED)
        total, bd = model(video, return_loss=True)
        ent = dict(perceptual_frames=seen[0].clone(), gen_frames=seen[-1].clone(), total=total.detach().float().clone(),
                   recon=bd.recon_loss.detach().float().clone(), aux=torch.as_tensor(bd.lfq_aux_loss).detach().float().clone(),
                   perceptual=bd.perceptual_loss.detach().float().clone(), gen=bd.adversarial_gen_loss.detach().float().clone(),
                   adaptive=torch.as_tensor(bd.adaptive_adversarial_weight).detach().float().clone())
        assert len(seen) == 3, len(seen)          # perceptual: real + recon frames (one draw), then the generator term's
        if digests:
            total.backward()
            ent["grads"] = {k: (grad_digest(p.grad.detach().float(), 256) if p.grad is not None else None)
                            for k, p in model.named_parameters() if not k.startswith("vgg.")}
        model.eval()
        torch.manual_seed(STEP_SEED)
        with torch.no_grad():
            total, bd = model(video, return_loss=True)
        ent["eval"] = dict(total=total.float().clone(), perceptual=bd.perceptual_loss.float().clone(),
                           gen=bd.adversarial_gen_loss.float().clone())
    finally:
        restore()
    return ent


def _standalone(vgg, dtype):
    x = _images(dtype).requires_grad_(True)
    feats = vgg(x)
    feats.float().sum().backward()
    return dict(features=feats.detach().float().clone(), grad_images=grad_digest(x.grad.detach().float(), 256))


def make(name):
    spec = VARIANTS[name]
    cfg = CONFIGS[BASE]
    kwargs = dict(cfg["kwargs"], use_gan=True, perceptual_loss_weight=0.1)
    ref = load_reference()
    video = W.synth_video(*cfg["video"][:3], cfg["video"][3], seed=cfg["vseed"])
    out = dict(name=name, kwargs=kwargs, vgg=dict(spec), vseed_vgg=VSEED, video_shape=tuple(cfg["video"]), wseed=cfg["wseed"],
               vseed=cfg["vseed"], iseed=ISEED, step_seed=STEP_SEED)
    model = _build(cfg, kwargs, spec)
    assert model.use_vgg and not any(k.startswith("vgg.") for k in model.state_dict())
    model.vgg.eval()
    out["standalone"] = _standalone(model.vgg, torch.float32)
    out["gen"] = _gen_step(model, video, ref)

    model16 = _build(cfg, kwargs, spec).bfloat16()
    model16.vgg.eval()
    out["bf16"] = dict(standalone=_standalone(model16.vgg, torch.bfloat16), gen=_gen_step(model16, video.bfloat16(), ref, digests=False))
    out["reference_commit"] = "a00519fa (v0.5.1)"
    out["third_party"] = "oracle/shims (restated LFQ/TaylorSeriesLinearAttn; real packages unavailable)"
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    torch.save(out, path)
    g = out["gen"]
    print(f"[golden] {name}: features {tuple(out['standalone']['features'].shape)}; total {g['total'].item():.6f} recon "
          f"{g['recon'].item():.6f} perceptual {g['perceptual'].item():.6f} gen {g['gen'].item():.6f} adaptive "
          f"{g['adaptive'].item():.6f}; bf16 total {out['bf16']['gen']['total'].item():.6f}; {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    for n in VARIANTS:
        make(n)
