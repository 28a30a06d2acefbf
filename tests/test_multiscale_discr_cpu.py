"""Multiscale discriminators (``multiscale_discrs=``, M:1085, M:1429-1441) on CPU: the flags against the reference's formula,
the checkpoint and copy surface, the refused configuration, and the multiscale losses, adaptive weights and discriminator
gradients of the restated oracle against the unmodified reference (tests/golden/mini_ms_*.pt,
oracle/make_multiscale_golden.py)."""
import itertools

import pytest
import torch
import torch.nn.functional as F

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from oracle.video_discr import SPECS, make_video_discrs
from tests.test_oracle import grad_digest_close
from tests.util import README_LAYERS, build_oracle, build_product, golden_video, load_golden

MINI = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS)
GOLDENS = ["mini_ms_gan", "mini_ms_gan_vgg", "mini_ms_vgg"]


def _pick(video, idx):
    return VideoTokenizer._pick_frames(video, idx)


@pytest.mark.parametrize("use_gan, ms_weight, n", list(itertools.product([True, False], [1., 0.5, 0.], [0, 1, 2])))
def test_flags_follow_reference_formula(use_gan, ms_weight, n):
    discrs = make_video_discrs()[:n]
    m = VideoTokenizer(**MINI, perceptual_loss_weight=0., use_gan=use_gan, multiscale_adversarial_loss_weight=ms_weight,
                       multiscale_discrs=tuple(discrs))
    assert m.has_multiscale_gan == (use_gan and ms_weight > 0.)                          # M:1431
    assert m.has_multiscale_discrs == (use_gan and ms_weight > 0. and n > 0)            # M:1437-1441
    assert isinstance(m.multiscale_discrs, torch.nn.ModuleList)
    assert [id(d) for d in m.multiscale_discrs] == [id(d) for d in discrs]              # held even when the flags are off


def test_parameters_checkpoint_and_copy_surface(tmp_path):
    m = VideoTokenizer(**MINI, perceptual_loss_weight=0., multiscale_discrs=tuple(make_video_discrs()))
    plain = VideoTokenizer(**MINI, perceptual_loss_weight=0.)
    ms_ids = {id(p) for p in m.multiscale_discrs.parameters()}
    # neither list holds them (M:1460-1474): the trainer builds their optimizers itself
    assert not ms_ids & {id(p) for p in m.parameters()} and not ms_ids & {id(p) for p in m.discr_parameters()}
    sd = m.state_dict()
    ms_keys = {k for k in sd if k.startswith("multiscale_discrs.")}
    assert ms_keys == {f"multiscale_discrs.{i}.{k}" for i in range(len(SPECS)) for k in make_video_discrs()[i].state_dict()}
    assert set(sd) - ms_keys == set(plain.state_dict())
    # strict loads: a model holding the modules loads their weights and misses none; one without drops them
    other = VideoTokenizer(**MINI, perceptual_loss_weight=0., multiscale_discrs=tuple(make_video_discrs(seed=9)))
    other.load_state_dict(sd)
    assert all(torch.equal(a, b) for a, b in zip(other.multiscale_discrs.parameters(), m.multiscale_discrs.parameters()))
    with pytest.raises(RuntimeError, match="Missing"):
        other.load_state_dict({k: v for k, v in sd.items() if k != sorted(ms_keys)[0]})
    plain.load_state_dict(sd)
    m.load_state_dict(plain.state_dict(), strict=False)                                 # non-strict: the modules keep theirs
    # copy_for_eval drops them (M:1482) and leaves the original as it was
    c = m.copy_for_eval()
    assert len(c.multiscale_discrs) == 0 and not c.has_multiscale_discrs and not c.training
    assert not any(k.startswith("multiscale_discrs.") for k in c.state_dict())
    assert len(m.multiscale_discrs) == len(SPECS) and m.has_multiscale_discrs
    # the pickled config stores multiscale_discrs=(): init_and_load_from gives a model without them
    path = tmp_path / "tok.pt"
    m.save(path)
    m2 = VideoTokenizer.init_and_load_from(path)
    assert len(m2.multiscale_discrs) == 0 and not m2.has_multiscale_discrs and m2.has_multiscale_gan
    assert ms_keys <= set(torch.load(path, weights_only=False)["model_state_dict"])
    # .bfloat16() casts them like any submodule
    assert all(p.dtype == torch.bfloat16 for p in m.bfloat16().multiscale_discrs.parameters())


def test_neither_image_gan_nor_vgg_is_refused_at_the_call():
    m = VideoTokenizer(**MINI, perceptual_loss_weight=0., adversarial_loss_weight=0., multiscale_discrs=tuple(make_video_discrs()))
    assert m.has_multiscale_discrs and not m.has_gan and not m.use_vgg
    for train in (True, False):
        m.train(train)
        with pytest.raises(ValueError, match="frame pick"):
            m(torch.randn(2, 3, 9, 32, 32), return_loss=True)
    with pytest.raises(NotImplementedError, match="image discriminator"):               # the reference asserts has_gan (M:1732)
        m(torch.randn(2, 3, 9, 32, 32), return_discr_loss=True)


@pytest.mark.parametrize("name", GOLDENS)
def test_golden_draw_order_and_quirk(name):
    """The reference draws the perceptual pick, then the image-GAN pick, and nothing for the multiscale terms; its generator
    loop never calls the multiscale discriminators, so they get no gradient from the generator step, and every multiscale
    loss and weight is the same."""
    g = load_golden(name)
    gs = g["gen"]
    b, _, t = g["video_shape"][:3]
    torch.manual_seed(g["step_seed"])
    draws = [torch.randn((b, t)).topk(1, dim=-1).indices for _ in range(2)]
    # the reference's picks: target and recon frames of the perceptual term, then the image-GAN term's frames -- or, without
    # an image GAN, the perceptual frames once more for the multiscale terms (M:1849-1850)
    expect = [gs["perceptual_frames"]] * 2 if "perceptual_frames" in gs else []
    expect.append(gs["gen_frames"] if "gen_frames" in gs else gs["perceptual_frames"])
    assert len(gs["frames"]) == len(expect) and all(torch.equal(a, e) for a, e in zip(gs["frames"], expect))
    assert torch.equal(draws[0], gs.get("perceptual_frames", gs.get("gen_frames")))
    if "perceptual_frames" in gs and "gen_frames" in gs:
        assert torch.equal(draws[1], gs["gen_frames"])
    assert len(gs["ms_gen"]) == len(SPECS) and (gs["ms_gen"] == gs["ms_gen"][0]).all()
    assert (gs["ms_weights"] == gs["ms_weights"][0]).all()
    assert all(gs["grads"][k] is None for k in gs["grads"] if k.startswith("multiscale_discrs."))
    assert (g["gen"]["eval"]["ms_weights"] == 1.).all()


def _oracle_step(g, need_norms):
    """The reference's generator step restated on the oracle: the train-mode reconstruction, the picked frames and, for the
    adaptive weights, the last-layer gradient norms of the perceptual and multiscale losses."""
    kw = dict(g["kwargs"], use_gan=False, perceptual_loss_weight=0.)
    oracle = build_oracle(build_product(kw, g["wseed"]), kw)
    w = oracle.sd["conv_out.conv.weight"].requires_grad_(need_norms)
    video = golden_video(g)
    recon = oracle.loss_forward(video, train=True)["recon"]
    gs = g["gen"]
    frames = _pick(recon, gs.get("gen_frames", gs.get("perceptual_frames")))
    ms_loss = -frames.mean()                                                             # hinge_gen_loss (M:123-124)
    norms = None
    if need_norms:
        s = g["vgg"]
        vgg = synth_data.fill_vgg_(synth_data.build_vgg(s["cfg"], s["hidden"], s["num_classes"]), g["vseed_vgg"]).eval()
        pf = gs["perceptual_frames"]
        perc = F.mse_loss(vgg(_pick(video, pf)), vgg(_pick(recon, pf)))
        norm_p = torch.autograd.grad(perc, w, retain_graph=True)[0].norm(p=2)
        norm_ms = torch.autograd.grad(ms_loss, w, retain_graph=True)[0].norm(p=2)
        norms = (norm_p, norm_ms)
    return video, recon.detach(), ms_loss.detach(), norms


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_multiscale_losses_match_reference(name):
    g = load_golden(name)
    gs = g["gen"]
    video, recon, ms_loss, norms = _oracle_step(g, "vgg" in g)
    for k in range(len(SPECS)):
        assert abs(ms_loss.item() - gs["ms_gen"][k].item()) < 1e-5, (k, ms_loss.item(), gs["ms_gen"])
    if norms is None:
        assert (gs["ms_weights"] == 1.).all()
    else:
        w = (norms[0] / norms[1].clamp(min=1e-5)).clamp(max=1e3)                         # M:1861-1866
        assert (abs(w.item() / gs["ms_weights"] - 1) < 1e-4).all(), (w.item(), gs["ms_weights"])
    if "discr" not in g:
        return
    gd = g["discr"]
    discrs = make_video_discrs(video.shape[1], g["mseed"])
    losses = [(F.relu(1 + d(recon)) + F.relu(1 - d(video))).mean() for d in discrs]    # M:1752-1762
    for got, ref in zip(losses, gd["ms_discr"]):
        assert abs(got.item() - ref.item()) < 1e-5 * max(1., abs(ref.item())), (got.item(), ref.item())
    (sum(losses) * g["kwargs"]["multiscale_adversarial_loss_weight"]).backward()         # the attribute weight (M:1776-1779)
    for i, d in enumerate(discrs):
        for k, p in d.named_parameters():
            grad_digest_close(p.grad, gd["grads"][f"multiscale_discrs.{i}.{k}"], 1e-4, k)
