"""TEST INFRASTRUCTURE ONLY.  fp16 fixtures: the UNMODIFIED reference run as ``model.half()`` on CPU, with the
protocol of the bf16 fixtures in oracle/make_golden.py: the same config, synthetic-weight seed and video seed as the
fp32 fixture named by ``codes_from``; tokenize stores the fp16 reference's own codes and pre-sign values, decode runs
on the fp32 fixture's codes so that both dtypes decode identical tokens, and the layer taps are strided samples of the
reference's own module outputs.  The fp16 path of the product is judged against the reference's OWN fp16 deviation
from fp32 (tests/test_f16_gpu.py).

    python -m oracle.make_f16_golden [names...]
"""
from __future__ import annotations

import os
import sys
import time

import torch

from oracle import weights as W
from oracle.make_golden import CONFIGS as FP32_CONFIGS, GOLDEN_DIR, _sample
from oracle.ref_loader import build_reference_tokenizer

# name -> the fp32 fixture whose config, seeds and codes it shares
CONFIGS = {"mini_f16": "mini", "readme_f16": "readme", "fsq_f16": "fsq", "mini_gateloop_f16": "mini_gateloop"}


def make(name: str):
    base = CONFIGS[name]
    cfg = FP32_CONFIGS[base]
    kwargs = dict(cfg["kwargs"])
    torch.manual_seed(0)
    model = build_reference_tokenizer(**kwargs)
    W.fill_state_dict_(model, cfg["wseed"])
    model.eval()
    video = W.synth_video(*cfg["video"][:3], cfg["video"][3], seed=cfg["vseed"])
    model = model.half()
    video = video.half()
    cs, ss = cfg.get("cs", 7), cfg.get("ss", 5)

    taps, hooks, presign = {}, [], {}

    def tap(nm):
        def fn(mod, inp, out):
            taps[nm] = _sample(out.detach().float(), cs, ss)
        return fn

    hooks.append(model.conv_in.register_forward_hook(tap("conv_in")))
    for i in range(len(kwargs["layers"])):
        hooks.append(model.encoder_layers[i].register_forward_hook(tap(f"enc{i}")))
        hooks.append(model.decoder_layers[i].register_forward_hook(tap(f"dec{i}")))
    hooks.append(model.quantizers.project_in.register_forward_hook(lambda m, i, o: presign.__setitem__("proj", o.detach().clone())))

    t0 = time.time()
    with torch.no_grad():
        codes = model.tokenize(video)
        t1 = time.time()
        codes_dec = torch.load(os.path.join(GOLDEN_DIR, base + ".pt"), weights_only=False)["codes"]
        recon = model.decode_from_code_indices(codes_dec).float()
        t2 = time.time()
    for h in hooks:
        h.remove()

    proj = presign["proj"].float()
    pre = proj if kwargs.get("use_fsq", False) else (proj / 10.).tanh() * 10.
    rs = cfg.get("rs", 4)
    out = dict(
        name=name, kwargs=kwargs, video_shape=tuple(cfg["video"]), wseed=cfg["wseed"], vseed=cfg["vseed"],
        codes=codes.clone(), presign=pre.clone(), taps=taps, tap_strides=(cs, ss),
        recon_sample=recon[:, :, :, ::rs, ::rs].contiguous().clone(), recon_stride=rs,
        recon_mean=recon.mean(dim=(3, 4)).clone(),
        ref_seconds=dict(tokenize=t1 - t0, decode=t2 - t1), torch_version=torch.__version__, cond=None,
        dtype="f16", codes_decoded=codes_dec.clone(), first_frame=True, codes_from=base,
        reference_commit="a00519fa (v0.5.1)",
        third_party="oracle/shims (restated LFQ/FSQ/TaylorSeriesLinearAttn; real packages unavailable)",
    )
    if cfg["full"]:
        out["recon"] = recon.clone()
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    torch.save(out, path)
    print(f"[golden] {name}: codes {tuple(codes.shape)}, min|presign|={pre.abs().min().item():.3e}, "
          f"recon absmax={recon.abs().max().item():.3f} finite={bool(torch.isfinite(recon).all())}, "
          f"tokenize {t1 - t0:.2f}s decode {t2 - t1:.2f}s, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    for n in sys.argv[1:] or list(CONFIGS):
        make(n)
