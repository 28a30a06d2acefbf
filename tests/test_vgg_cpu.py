"""The perceptual (VGG) loss on CPU (vgg.py): the construction rule, the checkpoint surface, the host repacks against torch's
formulation, and the torch restatement against the unmodified reference (tests/golden/mini_vgg16.pt, mini_vgg_narrow.pt)."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200 import vgg as V
from tests.test_oracle import grad_digest_close
from tests.util import README_LAYERS, load_golden

MINI = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, layers=README_LAYERS)
NARROW = (16, "M", 32, "M", 64, 64, "M")
GOLDENS = ["mini_vgg16", "mini_vgg_narrow"]


def _vgg(g):
    s = g["vgg"]
    return synth_data.fill_vgg_(synth_data.build_vgg(s["cfg"], s["hidden"], s["num_classes"]), g["vseed_vgg"])


def _images(g):
    return torch.randn(2, 3, 32, 32, generator=torch.Generator(device="cpu").manual_seed(g["iseed"]))


def test_construction_rule():
    vgg = synth_data.build_vgg(NARROW, 32)
    m = VideoTokenizer(**MINI, vgg=vgg)
    assert m.use_vgg and m.vgg is vgg and m.has_gan and m.discr is not None
    no_gan = VideoTokenizer(**MINI, vgg=vgg, use_gan=False)
    assert no_gan.use_vgg and no_gan.discr is None and not no_gan.has_gan
    for kw in (dict(perceptual_loss_weight=0.), dict(channels=2)):        # the reference builds no VGG here (M:1392)
        other = VideoTokenizer(**dict(MINI, **kw), vgg=vgg)
        assert not other.use_vgg and other.vgg is None
    default = VideoTokenizer(**MINI)                                      # vgg=None: unchanged
    assert default.vgg is None and not default.use_vgg and default.discr is None
    with pytest.raises(NotImplementedError):
        default(torch.randn(1, 3, 9, 32, 32), return_loss=True)
    with pytest.raises(NotImplementedError):
        default(torch.randn(1, 3, 9, 32, 32), return_discr_loss=True)


@pytest.mark.parametrize("edit, match", [
    (lambda v: v.features.insert(1, nn.BatchNorm2d(16)), "BatchNorm2d"),             # vgg*_bn
    (lambda v: v.features.__setitem__(0, nn.Conv2d(3, 16, 5, padding=2)), "features.0"),
    (lambda v: v.features.__setitem__(2, nn.AvgPool2d(2, 2)), "AvgPool2d"),
    (lambda v: v.features.__setitem__(2, nn.MaxPool2d(2, 2, ceil_mode=True)), "features.2"),
    (lambda v: setattr(v, "avgpool", nn.AdaptiveMaxPool2d(7)), "AdaptiveMaxPool2d"),
    (lambda v: v.classifier.insert(0, nn.Dropout()), "classifier.0"),
    (lambda v: v.classifier.append(nn.Softmax(dim=-1)), "Softmax"),
])
def test_unsupported_layouts_raise(edit, match):
    vgg = synth_data.build_vgg(NARROW, 32)
    edit(vgg)
    with pytest.raises(NotImplementedError, match=match):
        VideoTokenizer(**MINI, vgg=vgg)


def test_checkpoint_and_copy_surface(tmp_path):
    vgg = synth_data.build_vgg(NARROW, 32)
    m = VideoTokenizer(**MINI, vgg=vgg)
    ref = VideoTokenizer(**MINI, perceptual_loss_weight=0.)
    order = [k for k, _ in m.named_parameters()]
    sd = m.state_dict()
    assert not any(k.startswith("vgg.") for k in sd) and set(sd) == set(ref.state_dict())
    outer = nn.Sequential(m)                                                    # as a submodule: its prefix is honoured
    assert set(outer.state_dict()) == {"0." + k for k in sd}
    assert [tuple(p.shape) for p in m.parameters()] == [tuple(p.shape) for p in ref.parameters()]
    assert [id(p) for p in m.discr_parameters()] == [id(p) for p in m.discr.parameters()]
    full = dict(sd, **{"vgg." + k: v for k, v in vgg.state_dict().items()})      # a reference-style dict with VGG weights
    w0 = vgg.features[0].weight.detach().clone()
    m.load_state_dict(full)
    m.load_state_dict(sd)                                                      # strict: the VGG's own weights stand in
    assert m.vgg is vgg and torch.equal(vgg.features[0].weight, w0)
    assert [k for k, _ in m.named_parameters()] == order                     # the module tree is left as it was
    c = m.copy_for_eval()
    assert c.vgg is None and not c.use_vgg and m.vgg is vgg and not c.training
    assert not any(k.startswith("vgg.") for k, _ in c.named_parameters())
    path = tmp_path / "tok.pt"
    m.save(path)
    m2 = VideoTokenizer.init_and_load_from(path)                               # the pickled config stores vgg=None
    assert m2.vgg is None and not m2.use_vgg and m2.discr is None


@pytest.mark.parametrize("fmap", [(1, 1), (2, 2), (4, 4), (5, 5), (3, 9)])
def test_avgpool_fold_matches_adaptive_pool_then_linear(fmap):
    gen = torch.Generator(device="cpu").manual_seed(sum(fmap))
    C, O = 6, 10
    lin = nn.Linear(C * 49, O)
    x = torch.randn(3, C, *fmap, generator=gen)
    ref = lin(F.adaptive_avg_pool2d(x, (7, 7)).flatten(1))
    wf = V.fold_avgpool_linear(lin.weight, C, fmap, (7, 7))
    torch.testing.assert_close(F.conv2d(x, wf, lin.bias).flatten(1), ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_first_conv_channel_fold_matches_reference_repeat_and_slice(channels):
    gen = torch.Generator(device="cpu").manual_seed(channels)
    w, b = torch.randn(8, 3, 3, 3, generator=gen), torch.randn(8, generator=gen)
    x = torch.randn(2, channels, 10, 10, generator=gen)
    x3 = x.repeat(1, 3, 1, 1) if channels == 1 else x[:, :3]                 # M:1797-1803
    ref = F.conv2d(x3, w, b, padding=1)
    torch.testing.assert_close(F.conv2d(x, V.first_conv_weight(w, channels), b, padding=1), ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", GOLDENS)
def test_torch_restatement_matches_reference(name):
    g = load_golden(name)
    vgg = _vgg(g).eval()
    x = _images(g).requires_grad_(True)
    feats = V.vgg_torch(vgg, x)
    torch.testing.assert_close(feats.detach(), g["standalone"]["features"], rtol=1e-5, atol=1e-5)
    feats.sum().backward()
    grad_digest_close(x.grad, g["standalone"]["grad_images"], 1e-4, "images")


@pytest.mark.parametrize("name", GOLDENS)
def test_seeded_frame_choice_matches_reference(name):
    g = load_golden(name)
    b, _, t = g["video_shape"][:3]
    torch.manual_seed(g["step_seed"])
    assert torch.equal(torch.randn((b, t)).topk(1, dim=-1).indices, g["gen"]["perceptual_frames"])     # M:1792 first ...
    assert torch.equal(torch.randn((b, t)).topk(1, dim=-1).indices, g["gen"]["gen_frames"])            # ... then M:1827


def test_build_vgg_matches_torchvision_layout():
    tv = pytest.importorskip("torchvision")
    ours = synth_data.build_vgg(synth_data.VGG16_CFG, 4096, num_classes=1000)
    ref = tv.models.vgg16()
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    V.check_vgg(ref)
    ref.classifier = nn.Sequential(*ref.classifier[:-2])                     # the reference's default truncation (M:1403)
    V.check_vgg(ref)
    with pytest.raises(NotImplementedError, match="BatchNorm2d"):
        V.check_vgg(tv.models.vgg11_bn())


def test_cpu_resident_vgg_raises():
    g = load_golden("mini_vgg_narrow")
    with pytest.raises(RuntimeError, match="CUDA"):
        V.perceptual_loss(_vgg(g), _images(g), _images(g))
