"""Deterministic synthetic weights (keyed by ``state_dict`` name + shape) and videos for tests and bench.py.
Neutral data-synthesis helper: it imports neither the product package nor ``oracle/``.

The reference ships no checkpoints and the README-size generator has 117.8 M
parameters (470 MB fp32), far too large to commit.  Instead every test / bench
fills a model's generator tensors from a per-key seeded generator, so the
reference (in this container), the restated oracle and the CUDA product (on
the GPU box) all see bit-identical weights without shipping them.

The fill also de-degenerates the reference's default init (SURVEY.md 4 item 8):
``SqueezeExcite`` zero-inits its last conv with bias -10 (reference
magvit2_pytorch.py:218-219) which makes every ResidualUnit ~identity and would
hide conv errors; the up-samplers use a repeated-kernel init (M:829-836,
M:866-873).  Here every weight is i.i.d. normal with fan-in scaling.
"""
from __future__ import annotations

import hashlib

import torch


def _seed_for(key: str, seed: int) -> int:
    h = hashlib.sha256(f"{seed}:{key}".encode()).digest()
    return int.from_bytes(h[:8], "little") & 0x7FFFFFFFFFFFFFFF


def synth_tensor(key: str, shape, seed: int = 0, dtype=torch.float32) -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(_seed_for(key, seed))
    shape = tuple(shape)
    t = torch.randn(shape, generator=g, dtype=torch.float32)
    leaf = key.rsplit(".", 1)[-1]
    if leaf == "gamma":
        t = 1.0 + 0.1 * t
    elif leaf == "mem_kv":
        pass  # reference init is randn (M:357)
    elif leaf == "bias":
        t = 0.05 * t
    elif leaf == "weight":
        if len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = t * (fan_in ** -0.5)
        else:  # 1-d weight (the dead LayerNorm)
            t = 1.0 + 0.1 * t
    return t.to(dtype)


def is_generator_key(key: str) -> bool:
    return not (key.startswith("discr.") or key.startswith("multiscale_discrs.") or key.startswith("vgg."))


@torch.no_grad()
def fill_state_dict_(module, seed: int = 0):
    """Overwrite every floating-point generator tensor of ``module`` in place."""
    sd = module.state_dict()
    for k, v in sd.items():
        if not is_generator_key(k) or not v.is_floating_point():
            continue
        v.copy_(synth_tensor(k, v.shape, seed).to(v.dtype))
    return module


@torch.no_grad()
def fill_discr_(module, seed: int = 0):
    """Overwrite every floating-point ``discr.*`` tensor (the GAN's image discriminator) of a tokenizer in place;
    ``fill_state_dict_`` leaves them alone so that the generator's weights do not depend on whether one is built."""
    for k, v in module.state_dict().items():
        if k.startswith("discr.") and v.is_floating_point():
            v.copy_(synth_tensor(k, v.shape, seed).to(v.dtype))
    return module


class Vgg(torch.nn.Module):
    """torchvision.models.VGG's forward: features, avgpool, flatten, classifier."""

    def __init__(self, features, avgpool, classifier):
        super().__init__()
        self.features, self.avgpool, self.classifier = features, avgpool, classifier

    def forward(self, x):
        return self.classifier(torch.flatten(self.avgpool(self.features(x)), 1))


# torchvision's VGG16 feature configuration: output channels of each 3x3 conv, "M" = MaxPool2d(2, 2)
VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")


def build_vgg(cfg, hidden, num_classes=None, dropout=0.5, avgpool=(7, 7)):
    """A pure ``torch.nn`` module with torchvision's VGG attribute layout (features / avgpool / classifier and their child
    indices), so that no test needs torchvision.  num_classes=None truncates the classifier as the reference does for its
    default VGG16 (M:1403: the last ReLU-less Linear and the Dropout before it are dropped); otherwise the full classifier."""
    from torch import nn

    layers, c = [], 3
    for v in cfg:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(c, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            c = v
    cls = [nn.Linear(c * avgpool[0] * avgpool[1], hidden), nn.ReLU(True), nn.Dropout(p=dropout),
           nn.Linear(hidden, hidden), nn.ReLU(True), nn.Dropout(p=dropout)]
    cls = cls[:-1] if num_classes is None else cls + [nn.Linear(hidden, num_classes)]
    return Vgg(nn.Sequential(*layers), nn.AdaptiveAvgPool2d(avgpool), nn.Sequential(*cls))


@torch.no_grad()
def fill_vgg_(vgg, seed: int = 0):
    """Overwrite a VGG's weights in place from per-key seeded generators: He scaling (sqrt(2 / fan_in)) keeps the activations'
    magnitude through the ReLU layers, so the features and the perceptual loss do not vanish."""
    for k, v in vgg.state_dict().items():
        t = synth_tensor("vgg." + k, v.shape, seed)
        if k.endswith("weight"):
            t = t * 2 ** 0.5
        v.copy_(t.to(v.dtype))
    return vgg


def synth_video(batch, channels, frames, size, seed=1234):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    return torch.randn(batch, channels, frames, size, size, generator=g)
