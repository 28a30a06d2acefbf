"""TEST INFRASTRUCTURE ONLY.  tests/golden/<config>_io_grad.pt: the UNMODIFIED reference (oracle/ref_loader.py, quantiser shims)
in fp32 on the CPU, differentiated through its ordinary entry points (M:1522-1649):

* ``decode(z, cond)`` with z (and cond) requiring grad, eval and train mode;
* ``decode_from_code_indices(codes, cond)`` in train mode;
* ``encode(video, cond)`` with the video (and cond) requiring grad, eval mode;
* ``encode(video, quantize=True, cond)`` with the video requiring grad, eval and train mode.

For each case, with a seeded cotangent R of the output: the loss (out * R).sum() and the gradient digests (grad_digest,
at most 64 samples) of every parameter (None where the reference leaves it None) and of each floating input.

Runs only where the reference tree is present:   python -m oracle.make_io_grad_golden
"""
from __future__ import annotations

import os

import torch

from oracle import weights as W
from oracle.make_golden import CONFIGS, GOLDEN_DIR
from oracle.make_train_golden import grad_digest
from oracle.ref_loader import build_reference_tokenizer

MAX_ELEMS = 64
CASES = ("decode_eval", "decode_train", "decode_codes_train", "encode_eval", "encode_q_eval", "encode_q_train")
NAMES = ("mini", "mini_cond", "mini_sff", "mini_fsq", "mini_gateloop", "pad_reflect", "mini_noff")


def _cotangent(shape, seed):
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    return torch.randn(shape, generator=gen)


def _digest(t):
    return None if t is None else grad_digest(t.detach(), MAX_ELEMS)


def _run_case(model, case, video, z, codes, cond, ff, seed):
    """-> dict(loss, grads {name: digest | None}, inputs {name: digest | None})"""
    model.train() if case.endswith("_train") else model.eval()
    for p in model.parameters():
        p.grad = None
    cond_ = None if cond is None else cond.clone().requires_grad_(True)
    kw = dict(cond=cond_, video_contains_first_frame=ff)
    inputs = {}
    if case.startswith("decode_codes"):
        out = model.decode_from_code_indices(codes, **kw)
    elif case.startswith("decode"):
        z_ = z.clone().requires_grad_(True)
        inputs["quantized"] = z_
        out = model.decode(z_, **kw)
    else:
        v_ = video.clone().requires_grad_(True)
        inputs["video"] = v_
        out = model.encode(v_, quantize=case.startswith("encode_q"), **kw)
        if isinstance(out, tuple):
            out = out[0]
    if cond_ is not None:
        inputs["cond"] = cond_
    r = _cotangent(out.shape, seed)
    loss = (out * r).sum()
    if loss.requires_grad:
        loss.backward()
    return dict(loss=loss.detach().clone(), out_shape=tuple(out.shape), cot_seed=seed,
                grads={k: _digest(p.grad) for k, p in model.named_parameters()},
                inputs={k: _digest(t.grad) for k, t in inputs.items()})


def make(base, out_dir=GOLDEN_DIR):
    cfg = CONFIGS[base]
    kwargs = dict(cfg["kwargs"], use_gan=False, perceptual_loss_weight=0.)
    ff = cfg.get("first_frame", True)
    torch.manual_seed(0)
    model = build_reference_tokenizer(**kwargs)
    W.fill_state_dict_(model, cfg["wseed"])
    video = W.synth_video(*cfg["video"][:3], cfg["video"][3], seed=cfg["vseed"])
    out = dict(name=f"{base}_io_grad", base=base, kwargs=kwargs, video_shape=tuple(cfg["video"]), wseed=cfg["wseed"],
               vseed=cfg["vseed"], first_frame=ff)
    cond = None
    if kwargs.get("dim_cond") is not None:
        gen = torch.Generator(device="cpu")
        gen.manual_seed(cfg["cseed"])
        cond = torch.randn(cfg["video"][0], kwargs["dim_cond"], generator=gen)
        out["cond"] = cond
    model.eval()
    with torch.no_grad():           # the latents and codes the decode cases start from: the reference's own
        z, codes = model.encode(video, quantize=True, cond=cond, video_contains_first_frame=ff)[:2]
    # z (eval mode) is project_out of the codes' values: only the codes are stored
    out["codes"] = codes.to(torch.int32).clone()
    out["cases"] = {case: _run_case(model, case, video, z, codes, cond, ff, seed=1000 + i) for i, case in enumerate(CASES)}
    out["reference_commit"] = "a00519fa (v0.5.1)"
    out["third_party"] = "oracle/shims (restated LFQ/TaylorSeriesLinearAttn; real packages unavailable)"
    path = os.path.join(out_dir, f"{base}_io_grad.pt")
    torch.save(out, path)
    summary = ", ".join(f"{c} {v['loss'].item():.4f} ({sum(g is not None for g in v['grads'].values())} grads)"
                        for c, v in out["cases"].items())
    print(f"[golden] {base}_io_grad: {summary}; {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    for name in NAMES:
        make(name)
