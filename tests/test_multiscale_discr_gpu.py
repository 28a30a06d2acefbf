"""Multiscale discriminators (``multiscale_discrs=``, M:1085, M:1429-1441, M:1752-1765, M:1846-1881) in the training steps
against the unmodified reference (tests/golden/mini_ms_gan.pt, mini_ms_gan_vgg.pt, mini_ms_vgg.pt,
oracle/make_multiscale_golden.py): the generator and discriminator steps in fp32 and against the reference's own bf16 run,
the unchanged frame draws and device path, where each loss weight applies, and the reference trainer's optimizer steps."""
import pytest
import torch

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200 import train as T
from oracle.video_discr import SPECS, make_video_discrs
from tests.test_oracle import grad_digest_close
from tests.util import golden_video, load_golden

pytestmark = pytest.mark.gpu
GOLDENS = ["mini_ms_gan", "mini_ms_gan_vgg", "mini_ms_vgg"]
GAN_GOLDENS = ["mini_ms_gan", "mini_ms_gan_vgg"]


@pytest.fixture(autouse=True)
def _no_tf32():
    """cuDNN (the tokenizer's weight gradients, the user's Conv3d discriminators) in true fp32; restored even when a test fails."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _model(g, dtype=torch.float32, multiscale=True):
    torch.manual_seed(0)
    vgg = None
    if "vgg" in g:
        s = g["vgg"]
        vgg = synth_data.fill_vgg_(synth_data.build_vgg(s["cfg"], s["hidden"], s["num_classes"]), g["vseed_vgg"])
    discrs = tuple(make_video_discrs(g["video_shape"][1], g["mseed"])) if multiscale else ()
    m = VideoTokenizer(**g["kwargs"], vgg=vgg, multiscale_discrs=discrs)
    synth_data.fill_state_dict_(m, g["wseed"])
    synth_data.fill_discr_(m, g["wseed"])
    return m.cuda().to(dtype)


def _zero(m):
    for _, p in m.named_parameters():
        p.grad = None


def _gen_step(m, g, video, **kw):
    m.train()
    if m.vgg is not None:
        m.vgg.eval()
    _zero(m)
    torch.manual_seed(g["step_seed"])
    return m(video, return_loss=True, **kw)


def _discr_step(m, g, video, gp, **kw):
    m.train()
    _zero(m)
    torch.manual_seed(g["step_seed"])
    return m(video, return_discr_loss=True, apply_gradient_penalty=gp, **kw)


def _close(got, ref, rtol=1e-5):
    got, ref = float(torch.as_tensor(got).detach()), float(ref)
    assert abs(got - ref) < rtol * max(1., abs(ref)), (got, ref)


def _check_grads(m, digests, what):
    named = dict(m.named_parameters())
    gnorm = sum(d["norm"] ** 2 for d in digests.values() if d is not None) ** 0.5
    worst = 0.
    for k, dg in digests.items():
        p = named.get(k)
        if p is None:                       # the reference's always-built image discriminator, unused without the GAN term
            assert dg is None, (what, k)
            continue
        if dg is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, (what, k)
            continue
        assert p.grad is not None, (what, k)
        worst = max(worst, grad_digest_close(p.grad, dg, 5e-3, f"{what}:{k}", atol=1e-7 * gnorm))
    return worst


@pytest.mark.parametrize("name", GOLDENS)
def test_fp32_generator_step_vs_reference(name):
    g = load_golden(name)
    gs = g["gen"]
    m = _model(g)
    video = golden_video(g).cuda()
    total, bd = _gen_step(m, g, video)
    for got, key in ((total, "total"), (bd.recon_loss, "recon"), (bd.lfq_aux_loss, "aux"), (bd.perceptual_loss, "perceptual"),
                     (bd.adversarial_gen_loss, "gen")):
        _close(got, gs[key])
    _close(bd.adaptive_adversarial_weight, gs["adaptive"], 1e-4)
    assert len(bd.multiscale_gen_losses) == len(bd.multiscale_gen_adaptive_weights) == len(SPECS)
    for k in range(len(SPECS)):
        _close(bd.multiscale_gen_losses[k], gs["ms_gen"][k])
        _close(bd.multiscale_gen_adaptive_weights[k], gs["ms_weights"][k], 1e-4)
    total.backward()
    worst = _check_grads(m, gs["grads"], name)
    assert all(p.grad is None for p in m.multiscale_discrs.parameters())     # never called by the generator step (M:1852)
    print(f"{name}: {len(gs['grads'])} gradients, worst relative deviation {worst:.2e}; multiscale weights "
          f"{[float(w) for w in bd.multiscale_gen_adaptive_weights]}")
    m.eval()
    torch.manual_seed(g["step_seed"])
    with torch.no_grad():
        total, bd = m(video, return_loss=True)
    ev = gs["eval"]
    for got, key in ((total, "total"), (bd.perceptual_loss, "perceptual"), (bd.adversarial_gen_loss, "gen")):
        _close(got, ev[key])
    for k in range(len(SPECS)):
        _close(bd.multiscale_gen_losses[k], ev["ms_gen"][k])
    assert bd.multiscale_gen_adaptive_weights == [1.] * len(SPECS)


@pytest.mark.parametrize("name", GAN_GOLDENS)
def test_fp32_discriminator_step_vs_reference(name):
    g = load_golden(name)
    gd = g["discr"]
    m = _model(g)
    total, bd = _discr_step(m, g, golden_video(g).cuda(), True)
    for got, key in ((total, "total"), (bd.discr_loss, "hinge"), (bd.gradient_penalty, "penalty")):
        _close(got, gd[key])
    assert len(bd.multiscale_discr_losses) == len(SPECS)
    for got, ref in zip(bd.multiscale_discr_losses, gd["ms_discr"]):
        _close(got, ref)
    total.backward()
    worst = _check_grads(m, gd["grads"], name)
    assert all(p.grad is None for p in m.parameters())
    print(f"{name}: {len(gd['grads'])} discriminator gradients, worst relative deviation {worst:.2e}")


@pytest.mark.parametrize("name", GOLDENS)
def test_bf16_within_reference_bf16_error_budget(name):
    g = load_golden(name)
    g16 = g["bf16"]
    m = _model(g, torch.bfloat16)
    video = golden_video(g).cuda().bfloat16()
    total, bd = _gen_step(m, g, video)
    pairs = [(total, g16["gen"]["total"], g["gen"]["total"])]
    pairs += [(l, r16, r32) for l, r16, r32 in zip(bd.multiscale_gen_losses, g16["gen"]["ms_gen"], g["gen"]["ms_gen"])]
    pairs += [(w, r16, r32) for w, r16, r32 in zip(bd.multiscale_gen_adaptive_weights, g16["gen"]["ms_weights"],
                                                    g["gen"]["ms_weights"])]
    total.backward()
    assert torch.isfinite(m.conv_out.conv.weight.grad.float()).all()
    if "discr" in g:
        total, bd = _discr_step(m, g, video, False)
        # the fp32 golden's step has the penalty on, the bf16 one off: the fp32 total without it
        ref32 = g["discr"]["total"] - m.grad_penalty_loss_weight * g["discr"]["penalty"]
        pairs += [(total, g16["discr"]["total"], ref32)]
        pairs += [(l, r16, r32) for l, r16, r32 in zip(bd.multiscale_discr_losses, g16["discr"]["ms_discr"], g["discr"]["ms_discr"])]
    # as test_gan_gpu / test_vgg_gpu: the step's scalars carry the bf16 tokenizer's reconstruction, whose roundings differ
    # from the reference's, held to 3x the reference's own bf16 error
    for i, (got, ref16, ref32) in enumerate(pairs):
        got, ref16, ref32 = float(got), ref16.item(), ref32.item()
        e_prod, e_ref = abs(got - ref32), abs(ref16 - ref32)
        print(f"{name} pair {i}: product {got:.6f} err {e_prod:.3e}; reference bf16 err {e_ref:.3e}")
        assert e_prod <= 3.0 * e_ref + 1e-3 * max(1., abs(ref32)), (i, got, ref16, ref32)


def _recorded_picks(monkeypatch):
    seen = []
    pick = VideoTokenizer._pick_frames

    def recording(video, frame_indices):
        seen.append(frame_indices.clone())
        return pick(video, frame_indices)

    monkeypatch.setattr(VideoTokenizer, "_pick_frames", staticmethod(recording))
    return seen


@pytest.mark.parametrize("name", GOLDENS)
def test_draws_and_existing_terms_unchanged_by_multiscale_discrs(name, monkeypatch):
    """The multiscale terms draw nothing: the perceptual and image-discriminator picks, and every existing term, are those of
    the same model without multiscale discriminators; the total differs by the weighted multiscale sum alone."""
    g = load_golden(name)
    video = golden_video(g).cuda()
    seen = _recorded_picks(monkeypatch)
    out = {}
    for ms in (False, True):
        seen.clear()
        total, bd = _gen_step(_model(g, multiscale=ms), g, video)
        out[ms] = (total.detach(), bd, list(seen))
    (t0, b0, s0), (t1, b1, s1) = out[False], out[True]
    assert b0.multiscale_gen_losses == [] and b0.multiscale_gen_adaptive_weights == []
    # without multiscale discriminators: the perceptual pick (target and recon frames) and the image-GAN pick; with them one
    # more pick of the same frames for the multiscale terms (the image-GAN's, or the perceptual one's without an image GAN)
    assert len(s1) == len(s0) + 1 and all(torch.equal(a, b) for a, b in zip(s0, s1))
    assert torch.equal(s1[-1], s0[-1])
    for key in ("recon_loss", "lfq_aux_loss", "perceptual_loss", "adversarial_gen_loss", "adaptive_adversarial_weight"):
        _close(getattr(b1, key), getattr(b0, key), 1e-6)
    ms = sum(float(l) * float(w) for l, w in zip(b1.multiscale_gen_losses, b1.multiscale_gen_adaptive_weights))
    _close(t1, float(t0) + ms * g["kwargs"]["multiscale_adversarial_loss_weight"], 1e-5)


def test_call_site_weight_scales_generator_total_and_attribute_scales_discriminator_total():
    g = load_golden("mini_ms_gan")
    m = _model(g)
    video = golden_video(g).cuda()
    totals = {}
    for w in (None, 0., 2.):
        total, bd = _gen_step(m, g, video, multiscale_adversarial_loss_weight=w)
        totals[w] = float(total)
        ms = sum(float(l) * float(wt) for l, wt in zip(bd.multiscale_gen_losses, bd.multiscale_gen_adaptive_weights))
    attr = m.multiscale_adversarial_loss_weight
    assert attr == g["kwargs"]["multiscale_adversarial_loss_weight"] != 1.
    _close(totals[None], totals[0.] + attr * ms)
    _close(totals[2.], totals[0.] + 2. * ms)
    with torch.no_grad():
        base, bd = _discr_step(m, g, video, False)
        ignored, _ = _discr_step(m, g, video, False, multiscale_adversarial_loss_weight=7.)
        _close(ignored, base)                                   # the discriminator total uses the attribute (M:1776-1779)
        m.multiscale_adversarial_loss_weight = 2.
        scaled, _ = _discr_step(m, g, video, False)
    _close(scaled, float(base) + (2. - attr) * sum(float(x) for x in bd.multiscale_discr_losses))


def test_no_grad_paths_use_unit_weights():
    g = load_golden("mini_ms_gan")
    m = _model(g)
    video = golden_video(g).cuda()
    for train in (True, False):
        m.train(train)
        torch.manual_seed(g["step_seed"])
        with torch.no_grad():
            total, bd = m(video, return_loss=True)
        assert bd.multiscale_gen_adaptive_weights == [1.] * len(SPECS) and torch.isfinite(total)
        _close(bd.multiscale_gen_losses[0], g["gen"]["ms_gen"][0])
    # with a VGG the train-mode weights are ratios of gradient norms: the reference fails without gradients (M:1817-1820)
    v = load_golden("mini_ms_vgg")
    mv = _model(v).train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="gradients"):
        mv(golden_video(v).cuda(), return_loss=True)


def test_uint8_video_reaches_the_multiscale_discriminators_as_model_dtype_fraction():
    g = load_golden("mini_ms_gan")
    m = _model(g, torch.bfloat16)
    seen = []
    for d in m.multiscale_discrs:
        d.register_forward_pre_hook(lambda mod, args: seen.append(args[0]))
    video = (golden_video(g).clamp(-2, 2) * 60 + 128).to(torch.uint8).cuda()
    with torch.no_grad():
        _discr_step(m, g, video, False)
    real = seen[0]
    assert real.dtype == torch.bfloat16 and torch.equal(real, (video.float() / 255.).bfloat16())
    assert seen[1].dtype == torch.bfloat16 and seen[1].shape == video.shape


def test_reference_trainer_steps_bf16():
    """Two iterations of the reference trainer's step with multiscale discriminators (T:339-446): generator step and AdamW;
    then the discriminator step, backward, gradient clipping and one AdamW per multiscale module, which changes only that
    module's parameters."""
    g = load_golden("mini_ms_gan_vgg")
    m = _model(g, torch.bfloat16)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    dopt = torch.optim.AdamW(m.discr_parameters(), lr=1e-4)
    ms_opts = [torch.optim.AdamW(d.parameters(), lr=1e-3) for d in m.multiscale_discrs]
    video = golden_video(g).cuda().bfloat16()
    m.train()
    m.vgg.eval()
    for step in range(2):
        opt.zero_grad()
        loss, bd = m(video, return_loss=True)
        loss.backward()
        opt.step()
        opt.zero_grad()
        dopt.zero_grad()
        for o in ms_opts:
            o.zero_grad()
        gen_before = [p.detach().clone() for p in m.parameters()]
        dloss, dbd = m(video, return_discr_loss=True, apply_gradient_penalty=step == 0)
        dloss.backward()
        assert all(p.grad is None for p in m.parameters())
        assert all(p.grad is not None for p in m.multiscale_discrs.parameters())
        torch.nn.utils.clip_grad_norm_(m.discr_parameters(), 1.)
        for d in m.multiscale_discrs:
            torch.nn.utils.clip_grad_norm_(d.parameters(), 1.)
        dopt.step()
        for i, o in enumerate(ms_opts):
            before = {k: p.detach().clone() for k, p in m.named_parameters()}
            o.step()
            changed = {k for k, p in m.named_parameters() if not torch.equal(before[k], p)}
            assert changed and all(k.startswith(f"multiscale_discrs.{i}.") for k in changed), (step, i, changed)
        assert all(torch.equal(a, p) for a, p in zip(gen_before, m.parameters()))
        for v in (loss, dloss, *bd.multiscale_gen_losses, *bd.multiscale_gen_adaptive_weights, *dbd.multiscale_discr_losses):
            assert torch.isfinite(torch.as_tensor(v).float()).all(), step


@pytest.mark.parametrize("name", GAN_GOLDENS)
def test_device_path_unchanged(name, monkeypatch):
    """A generator step (forward and backward) launches the same kernels with and without multiscale discriminators, except
    that with a VGG the multiscale adaptive weight takes one more last-layer weight gradient."""
    g = load_golden(name)
    video = golden_video(g).cuda()
    extra = []
    llwg = T.TrainRunner.last_layer_weight_grad

    def counted(self, g_recon):
        n0 = self.eng.launches
        out = llwg(self, g_recon)
        extra.append(self.eng.launches - n0)
        return out

    monkeypatch.setattr(T.TrainRunner, "last_layer_weight_grad", counted)
    launches, calls = {}, {}
    for ms in (False, True):
        m = _model(g, multiscale=ms)
        _gen_step(m, g, video)[0].backward()                  # warm-up: engines, packs
        engines = [m.engine, m.discr._pack_cache.engine] + ([m._vgg_cache.engine] if m.vgg is not None else [])
        torch.cuda.synchronize()
        n0 = [e.launches for e in engines]
        extra.clear()
        _gen_step(m, g, video)[0].backward()
        torch.cuda.synchronize()
        launches[ms] = sum(e.launches - n for e, n in zip(engines, n0))
        calls[ms] = list(extra)
    assert len(calls[True]) == len(calls[False]) + (1 if "vgg" in g else 0)
    assert launches[True] == launches[False] + sum(calls[True][len(calls[False]):]), (launches, calls)
    print(f"{name}: {launches[False]} launches without, {launches[True]} with multiscale discriminators")
