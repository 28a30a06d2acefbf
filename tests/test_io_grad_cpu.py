"""Differentiable encode / decode / decode_from_code_indices without a GPU: the rule that picks the differentiable path, the
parameters each entry point reaches against the reference's gradients (tests/golden/*_io_grad.pt), and the fixtures'
regeneration by oracle/make_io_grad_golden.py where the reference tree is present."""
import itertools

import pytest
import torch

from magvit2_pytorch_b200.train import reached_parameters
from tests.util import build_product, load_golden

IO_GOLDENS = ["mini", "mini_cond", "mini_sff", "mini_fsq", "mini_gateloop", "pad_reflect", "mini_noff"]

# golden case -> (entry, train mode, quantize)
CASES = {"decode_eval": ("decode", False, False), "decode_train": ("decode", True, False),
         "decode_codes_train": ("decode_codes", True, False), "encode_eval": ("encode", False, False),
         "encode_q_eval": ("encode", False, True), "encode_q_train": ("encode", True, True)}


def _model():
    return build_product(dict(image_size=32, init_dim=16, max_dim=64, codebook_size=1024,
                              layers=("residual", "compress_space", "compress_time", "residual"), use_gan=False,
                              perceptual_loss_weight=0.))


@pytest.mark.parametrize("grad_mode,train,input_grad,frozen", list(itertools.product((True, False), repeat=4)))
def test_selection_rule_truth_table(grad_mode, train, input_grad, frozen):
    """The differentiable path is taken iff grad mode is on and either a floating input requires grad or, in train mode, a
    parameter the call reaches requires grad; otherwise None (the no-grad path).  `frozen`: every parameter frozen."""
    m = _model()
    m.train(train)
    for p in m.parameters():
        p.requires_grad_(not frozen)
    z = torch.zeros(1, m.quantizers.dim, 2, 4, 4, requires_grad=input_grad)
    with torch.set_grad_enabled(grad_mode):
        got_decode = m._grad_params((z, None), "decode", True, 5)
        got_codes = m._grad_params((None,), "decode_codes", True, 5)
    want = grad_mode and (input_grad or (train and not frozen))
    assert (got_decode is not None) == want
    assert (got_codes is not None) == (grad_mode and train and not frozen)      # codes are integers: never an input gradient
    if want:
        assert len(got_decode) == (0 if frozen else len(reached_parameters(m, "decode", True, 5)))


def test_frozen_parameters_are_not_handed_over():
    m = _model()
    m.train()
    for p in m.conv_out.parameters():
        p.requires_grad_(False)
    got = m._grad_params((None,), "decode", True, 5)
    assert got and not any(p is q for p in got for q in m.conv_out.parameters())


@pytest.mark.parametrize("name", IO_GOLDENS)
def test_reached_parameters_match_the_reference_gradients(name):
    """For every golden case, the parameters the entry point hands to the differentiable path are exactly those whose
    reference gradient is not None."""
    g = load_golden(f"{name}_io_grad")
    m = build_product(g["kwargs"], g["wseed"])
    ff = g["first_frame"]
    by_id = {id(p): k for k, p in m.named_parameters()}
    names = set(by_id.values())
    frames_in = g["video_shape"][2]
    frames_out = g["codes"].shape[1] * m.time_downsample_factor - (m.time_padding if ff else 0)
    for case, (entry, train, quantize) in CASES.items():
        m.train(train)
        frames = frames_in if entry == "encode" else frames_out
        got = {by_id[id(p)] for p in reached_parameters(m, entry, ff, frames, quantize)}
        want = {k for k, d in g["cases"][case]["grads"].items() if d is not None and k in names}
        assert got == want, (case, sorted(got ^ want))


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    return a == b


@pytest.mark.parametrize("name", IO_GOLDENS)
def test_goldens_regenerate_bit_for_bit(name, tmp_path):
    from oracle.ref_loader import reference_available
    if not reference_available():
        pytest.skip("the reference tree is not present")
    from oracle.make_io_grad_golden import make
    make(name, out_dir=str(tmp_path))
    new = torch.load(tmp_path / f"{name}_io_grad.pt", map_location="cpu", weights_only=False)
    assert _same(new, load_golden(f"{name}_io_grad"))
