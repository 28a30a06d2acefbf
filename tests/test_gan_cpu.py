"""The GAN discriminator (gan.py) on CPU: the construction rule, the checkpoint surface, the host repacks against the
reference's formulation, and the torch restatement against the unmodified reference (tests/golden/mini_gan.pt)."""
import pytest
import torch
import torch.nn.functional as F

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200 import gan
from tests.test_oracle import grad_digest_close
from tests.util import README_LAYERS, load_golden

MINI = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS)


def _gan_model(**kw):
    g = load_golden("mini_gan")
    torch.manual_seed(0)
    m = VideoTokenizer(**dict(g["kwargs"], **kw))
    synth_data.fill_state_dict_(m, g["wseed"])
    synth_data.fill_discr_(m, g["wseed"])
    return m, g


def _images(g):
    gen = torch.Generator(device="cpu").manual_seed(g["iseed"])
    return torch.randn(2, 3, 32, 32, generator=gen)


def test_discr_key_shapes_match_reference():
    m, g = _gan_model()
    assert m.has_gan and m.discr is not None
    got = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("discr.")}
    assert got == g["discr_shapes"]
    assert [id(p) for p in m.discr_parameters()] == [id(p) for p in m.discr.parameters()]


def test_construction_rule():
    default = VideoTokenizer(**MINI)                          # perceptual_loss_weight = 0.1: a VGG is configured
    assert default.discr is None and not default.has_gan and default.discr_parameters() == []
    with pytest.raises(NotImplementedError):
        default(torch.randn(1, 3, 9, 32, 32), return_loss=True)
    with pytest.raises(NotImplementedError):
        default(torch.randn(1, 3, 9, 32, 32), return_discr_loss=True)
    no_gan = VideoTokenizer(**MINI, use_gan=False, perceptual_loss_weight=0.)
    assert no_gan.discr is None and not no_gan.has_gan
    no_adv = VideoTokenizer(**MINI, perceptual_loss_weight=0., adversarial_loss_weight=0.)
    assert no_adv.discr is None and not no_adv.has_gan
    gan_m = VideoTokenizer(**MINI, perceptual_loss_weight=0.)
    assert gan_m.has_gan
    assert [tuple(p.shape) for p in gan_m.parameters()] == [tuple(p.shape) for p in no_gan.parameters()]   # generator only
    base = dict(dim=64, image_size=32, channels=3)
    with pytest.raises(NotImplementedError, match="filter3d"):
        VideoTokenizer(**MINI, perceptual_loss_weight=0., discr_kwargs=dict(base, antialiased_downsample=True))
    with pytest.raises(NotImplementedError, match="dim_head"):
        VideoTokenizer(**MINI, perceptual_loss_weight=0., discr_kwargs=dict(base, linear_attn_dim_head=16))
    custom = VideoTokenizer(**MINI, perceptual_loss_weight=0., discr_kwargs=dict(base, max_dim=256, ff_mult=2))
    assert custom.discr.blocks[-1][0].net[0].weight.shape[0] == 256


def test_save_load_roundtrip_carries_discr(tmp_path):
    m, _ = _gan_model()
    path = tmp_path / "tok.pt"
    m.save(path)
    m2 = VideoTokenizer.init_and_load_from(path)
    assert m2.has_gan
    sd, sd2 = m.state_dict(), m2.state_dict()
    keys = [k for k in sd if k.startswith("discr.")]
    assert keys and all(torch.equal(sd[k], sd2[k]) for k in keys)
    c = m.copy_for_eval()
    assert torch.equal(c.discr.to_logits[3].weight, m.discr.to_logits[3].weight)
    bad = {k: v for k, v in sd.items() if k != keys[0]}
    with pytest.raises(RuntimeError, match="Missing"):
        m2.load_state_dict(bad)


def test_host_repacks_match_reference_formulation():
    gen = torch.Generator(device="cpu").manual_seed(3)
    C, Co = 8, 12
    h = torch.randn(2, C, 8, 8, generator=gen)
    # downsample: 'b c (h p1) (w p2) -> b (c p1 p2) h w' + 1x1 conv == 2x2 stride-2 conv
    w = torch.randn(Co, 4 * C, 1, 1, generator=gen)
    b = torch.randn(Co, generator=gen)
    ref = F.conv2d(h.reshape(2, C, 4, 2, 4, 2).permute(0, 1, 3, 5, 2, 4).reshape(2, 4 * C, 4, 4), w, b)
    torch.testing.assert_close(F.conv2d(h, gan.unshuffle_conv_weight(w), b, stride=2), ref)
    # to_logits: Linear over the '(c h w)' flatten == a conv covering the feature map
    lin = torch.nn.Linear(C * 4 * 4, 1)
    x = torch.randn(3, C, 4, 4, generator=gen)
    torch.testing.assert_close(F.conv2d(x, gan.logits_conv_weight(lin, C, (4, 4)), lin.bias).reshape(-1), lin(x.flatten(1))[:, 0])
    # stride-2 data gradients == 1x1 convs into the depth-to-space store (reference order '(c p1 p2)')
    g = torch.randn(2, Co, 4, 4, generator=gen)
    for wd_fn, w_s2, k in ((gan.unshuffle_dgrad_weight, gan.unshuffle_conv_weight(w), 2),
                           (gan.stride2_1x1_dgrad_weight, torch.randn(Co, C, 1, 1, generator=gen), 1)):
        xr = torch.zeros(2, C, 8, 8, requires_grad=True)
        gx_ref, = torch.autograd.grad(F.conv2d(xr, w_s2, stride=2), xr, g)
        wd = wd_fn(w if k == 2 else w_s2)
        gx = F.pixel_shuffle(F.conv2d(g, wd), 2)
        torch.testing.assert_close(gx, gx_ref)


def test_torch_restatement_matches_reference():
    m, g = _gan_model()
    d = m.discr
    x = _images(g).requires_grad_(True)
    logits = gan.discriminator_torch(d, x)
    torch.testing.assert_close(logits.detach(), g["standalone"]["logits"], rtol=1e-5, atol=1e-6)
    logits.sum().backward()
    grad_digest_close(x.grad, g["standalone"]["grad_images"], 1e-4, "images")
    for k, p in d.named_parameters():
        grad_digest_close(p.grad, g["standalone"]["grads"][k], 1e-4, k, atol=1e-7)
        p.grad = None
    gp = gan.gradient_penalty(d, _images(g))
    torch.testing.assert_close(gp.detach(), g["penalty"]["value"], rtol=1e-5, atol=0)
    gp.backward()
    for k, p in d.named_parameters():
        if g["penalty"]["grads"][k] is None:        # the logit bias does not enter the input gradient
            assert p.grad is None or not p.grad.any(), k
            continue
        grad_digest_close(p.grad, g["penalty"]["grads"][k], 1e-4, k, atol=1e-7)


def test_seeded_frame_choice_matches_reference():
    g = load_golden("mini_gan")
    b, _, t = g["video_shape"][:3]
    for step in ("discr", "discr_gp", "gen"):
        torch.manual_seed(g["step_seed"])
        assert torch.equal(torch.randn((b, t)).topk(1, dim=-1).indices, g[step]["frames"]), step


def test_cpu_resident_discriminator_raises():
    m, g = _gan_model()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.discr(_images(g))
    with pytest.raises(RuntimeError):
        m(torch.randn(2, 3, 9, 32, 32), return_discr_loss=True)
