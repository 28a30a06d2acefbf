"""A small deterministic video discriminator for the multiscale-discriminator tests and goldens (reference
``multiscale_discrs``, M:1085, M:1752-1765): the reference takes any module mapping a whole (B, C, T, H, W) video to logits,
so this one is ours -- Conv3d, LeakyReLU, Conv3d, then the mean over (C, T, H, W) giving (B,).  The golden generator
(oracle/make_multiscale_golden.py) and the tests build theirs here, with weights filled from per-key seeded generators
(synth_data.synth_tensor), so both sides see bit-identical modules whatever torch's global seed is.
"""
from __future__ import annotations

import torch
from torch import nn

import synth_data

# (hidden channels, spatial stride of the first conv): two scales, as a user would pass them
SPECS = ((8, 1), (4, 2))


class VideoDiscriminator(nn.Module):
    def __init__(self, channels=3, dim=8, stride=1):
        super().__init__()
        self.conv1 = nn.Conv3d(channels, dim, 3, stride=(1, stride, stride), padding=1)
        self.act = nn.LeakyReLU(0.1)
        self.conv2 = nn.Conv3d(dim, 1, 3, padding=1)

    def forward(self, video):
        return self.conv2(self.act(self.conv1(video))).mean(dim=(1, 2, 3, 4))


@torch.no_grad()
def make_video_discrs(channels=3, seed=0, specs=SPECS):
    """One VideoDiscriminator per spec, weights keyed as the tokenizer's state_dict holds them (multiscale_discrs.<i>.*)."""
    discrs = []
    for i, (dim, stride) in enumerate(specs):
        d = VideoDiscriminator(channels, dim, stride)
        for k, v in d.state_dict().items():
            v.copy_(synth_data.synth_tensor(f"multiscale_discrs.{i}.{k}", v.shape, seed))
        discrs.append(d)
    return discrs
