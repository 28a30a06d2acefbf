"""Attention dropout without a GPU: the numpy Philox replica against Random123's known-answer vectors, the keep rule at its
edges, the constructor's rules and checkpoint round trip, the C ABI's declaration and binding, and the training restatement's
dropout step."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from magvit2_pytorch_b200 import VideoTokenizer, _lib
from magvit2_pytorch_b200.train import _softmax_attention, dropout_scale
from tests.attn_dropout_ref import dropout_scale as ref_scale
from tests.attn_dropout_ref import keep_mask, keep_threshold, philox4x32_10

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MINI = dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024, use_gan=False, perceptual_loss_weight=0.,
            layers=("residual", "compress_space", "attend_space", "compress_time", "attend_time"))


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32 with 10 rounds."""
    got = philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert tuple(int(w) for w in got) == want


def test_keep_threshold_at_the_edges():
    """keep iff word >= floor(p * 2^32) with p the fp32 value: the smallest p, one half and the largest fp32 below 1."""
    assert keep_threshold(2.0 ** -32) == 1 and keep_threshold(1e-12) == 0        # 1e-12 keeps every word
    assert keep_threshold(0.5) == 2 ** 31
    assert keep_threshold(1 - 2.0 ** -24) == 2 ** 32 - 2 ** 8
    assert keep_threshold(0.1) == int(np.floor(float(np.float32(0.1)) * 2.0 ** 32)) != int(0.1 * 2 ** 32)
    assert ref_scale(0.5) == 2.0 and ref_scale(1 - 2.0 ** -24) == 2.0 ** 24
    for p in (0.1, 0.2, 0.3, 1e-7, 1 - 2.0 ** -24):
        assert dropout_scale(p) == ref_scale(p), p


def test_keep_mask_layout_and_rule():
    """keep[seq][h][i][j] is word j & 3 of the counter (i, j >> 2, seq, h | call << 16) against the threshold."""
    seed, call, p = 0x0123456789ABCDEF, 3, 0.5
    m = keep_mask(seed, call, p, n_seq=3, heads=2, L=5, n_mem=4)
    assert m.shape == (3, 2, 5, 9) and m.dtype == np.uint8
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
    for s, h, i, j in ((0, 0, 0, 0), (2, 1, 4, 8), (1, 0, 3, 6), (2, 1, 0, 5)):
        w = philox4x32_10(np.array([i, j >> 2, s, h | call << 16], dtype=np.uint32), key)[j & 3]
        assert m[s, h, i, j] == (int(w) >= 2 ** 31)
    assert not np.array_equal(m, keep_mask(seed, call + 1, p, 3, 2, 5, 4))
    assert not np.array_equal(m, keep_mask(seed ^ (1 << 40), call, p, 3, 2, 5, 4))     # the seed's high word is part of the key


def test_constructor_rules_and_checkpoint_round_trip(tmp_path):
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            VideoTokenizer(**MINI, attn_dropout=bad)
    with pytest.raises(NotImplementedError, match="attn_dropout=1"):
        VideoTokenizer(**MINI, attn_dropout=1.)
    m = VideoTokenizer(**MINI, attn_dropout=0.1)
    assert m.attn_dropout == 0.1
    m.save(tmp_path / "tok.pt")
    back = VideoTokenizer.init_and_load_from(tmp_path / "tok.pt")
    assert back.attn_dropout == 0.1
    for (k, a), (_, b) in zip(m.state_dict().items(), back.state_dict().items()):
        assert torch.equal(a, b), k


def test_header_binding_and_struct_layout():
    """mv2_dropout_args is {uint64 seed; uint32 call; float p} (16 bytes); the two entry points are declared with the argument
    counts _lib binds."""
    src = open(os.path.join(ROOT, "include", "magvit2_b200.h")).read()
    body = re.search(r"typedef struct mv2_dropout_args \{(.*?)\} mv2_dropout_args;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert [ln.split() for ln in body.replace(";", "\n").splitlines() if ln.strip()] == [
        ["uint64_t", "seed"], ["uint32_t", "call"], ["float", "p"]]
    A = _lib.DropoutArgs
    assert ctypes.sizeof(A) == 16 and (A.seed.offset, A.call.offset, A.p.offset) == (0, 8, 12)
    for name in ("mv2_attention_dropout", "mv2_attention_dropout_mask"):
        decl = re.search(rf"int {name}\((.*?)\);", src, re.S).group(1)
        assert len(decl.split(",")) == len(_lib.SIGNATURES[name][1]), name
    a = A(seed=2 ** 64 - 1, call=65535, p=0.1)
    assert a.seed == 2 ** 64 - 1 and a.call == 65535 and a.p == float(np.float32(0.1))


def test_restatement_applies_keep_and_scale_after_the_softmax():
    """The training backward's restatement: attn * keep * fp32(1 / (1 - p)) after the softmax; all-ones keep scales the output,
    a dropped key leaves the denominator alone."""
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn((2, 3, 5, 8), generator=g, dtype=torch.float64) for _ in range(3))
    k, v = torch.cat((torch.randn((2, 3, 4, 8), generator=g, dtype=torch.float64), k), 2), torch.cat((torch.randn((2, 3, 4, 8), generator=g, dtype=torch.float64), v), 2)
    base = _softmax_attention(q, k, v, causal=True)
    ones = torch.ones((2, 3, 5, 9), dtype=torch.uint8)
    torch.testing.assert_close(_softmax_attention(q, k, v, True, (ones, 0.25)), base * dropout_scale(0.25), rtol=1e-12, atol=1e-14)
    keep = ones.clone()
    keep[..., 2] = 0
    w = (torch.einsum("bhid,bhjd->bhij", q, k) * 8 ** -0.5).masked_fill(torch.ones(5, 9, dtype=torch.bool).triu(5), -torch.inf).softmax(-1)
    want = torch.einsum("bhij,bhjd->bhid", w * keep * dropout_scale(0.5), v)
    torch.testing.assert_close(_softmax_attention(q, k, v, True, (keep, 0.5)), want, rtol=1e-12, atol=1e-14)
