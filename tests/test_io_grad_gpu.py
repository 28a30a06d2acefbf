"""Differentiable encode / decode / decode_from_code_indices on the device: fp32 losses and gradients against the unmodified
reference's autograd (tests/golden/*_io_grad.pt, oracle/make_io_grad_golden.py), bf16 against fp32, the video's gradient on the
engine's kernels (its float64 checks are tests/test_video_dgrad_gpu.py), and the no-grad path left as it was."""
import pytest
import torch
import torch.nn.functional as F

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.train import _code_values
from oracle.make_io_grad_golden import _cotangent
from tests.test_io_grad_cpu import CASES, IO_GOLDENS
from tests.test_oracle import grad_digest_close
from tests.util import build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu


def _require_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _latents(model, codes):
    """The reference's eval-mode encode(quantize=True) output: project_out of the codes' values (indices_to_codes)."""
    qz = model.quantizers
    vals = _code_values(codes.long(), qz, model.use_fsq)
    with torch.no_grad():
        z = F.linear(vals, qz.project_out.weight.float().cpu(), qz.project_out.bias.float().cpu())
    return z.permute(0, 4, 1, 2, 3).contiguous()


def _run(model, case, g, dev, dtype=torch.float32):
    """One golden case on the product -> (loss, output, {input name: tensor})."""
    entry, train, quantize = CASES[case]
    model.train(train)
    for p in model.parameters():
        p.grad = None
    ff = g["first_frame"]
    cond = g["cond"].to(dev).requires_grad_(True) if g.get("cond") is not None else None
    inputs = {} if cond is None else {"cond": cond}
    if entry == "decode_codes":
        out = model.decode_from_code_indices(g["codes"].long().to(dev), cond=cond, video_contains_first_frame=ff)
    elif entry == "decode":
        z = _latents(model, g["codes"]).to(dev, dtype).requires_grad_(True)
        inputs["quantized"] = z
        out = model.decode(z, cond=cond, video_contains_first_frame=ff)
    else:
        v = golden_video(g).to(dev, dtype).requires_grad_(True)
        inputs["video"] = v
        out = model.encode(v, quantize=quantize, cond=cond, video_contains_first_frame=ff)
        out = out[0] if quantize else out
    assert out.grad_fn is not None, case
    r = _cotangent(out.shape, g["cases"][case]["cot_seed"]).to(dev)
    loss = (out.float() * r).sum()
    loss.backward()
    return loss, out, inputs


@pytest.mark.parametrize("name", IO_GOLDENS)
def test_fp32_losses_and_gradients_vs_reference_golden(name):
    _require_cuda()
    g = load_golden(f"{name}_io_grad")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    named = dict(model.named_parameters())
    for case, ref in g["cases"].items():
        loss, out, inputs = _run(model, case, g, "cuda")
        scale = float((out.detach().float().abs() * _cotangent(out.shape, ref["cot_seed"]).cuda().abs()).sum())
        assert abs(loss.item() - ref["loss"].item()) <= 1e-5 * max(1.0, scale), (case, loss.item(), ref["loss"].item())
        gnorm = sum(d["norm"] ** 2 for d in ref["grads"].values() if d is not None) ** 0.5
        checked = 0
        for k, dg in ref["grads"].items():
            if k not in named:
                continue
            p = named[k]
            if dg is None:
                assert p.grad is None, (case, k)
                continue
            assert p.grad is not None, (case, k)
            grad_digest_close(p.grad, dg, 5e-3, (case, k), atol=1e-7 * gnorm)
            checked += 1
        for k, t in inputs.items():
            dg = ref["inputs"][k]
            if dg is None:
                assert t.grad is None or float(t.grad.abs().max()) == 0.0, (case, k)
            else:
                assert t.grad is not None, (case, k)
                grad_digest_close(t.grad, dg, 5e-3, (case, k), atol=1e-7 * dg["norm"])
        assert checked > 0, case


def _cos(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()).clamp(min=1e-300))


@pytest.mark.parametrize("name", ["mini", "mini_sff", "mini_cond"])
def test_bf16_gradients_agree_with_fp32(name):
    """Per side (parameters, inputs) the bf16 path's gradient points where the fp32 path's does."""
    _require_cuda()
    g = load_golden(f"{name}_io_grad")
    m32 = build_product(g["kwargs"], g["wseed"]).cuda()
    m16 = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    for case in ("decode_train", "encode_eval", "encode_q_train"):
        _, _, in32 = _run(m32, case, g, "cuda")
        _, _, in16 = _run(m16, case, g, "cuda", torch.bfloat16)
        p32 = torch.cat([p.grad.reshape(-1).float() for p in m32.parameters() if p.grad is not None])
        p16 = torch.cat([p.grad.reshape(-1).float() for p in m16.parameters() if p.grad is not None])
        assert _cos(p32, p16) > 0.99, (case, _cos(p32, p16))
        for k in in32:
            assert _cos(in32[k].grad, in16[k].grad.float()) > 0.99, (case, k, _cos(in32[k].grad, in16[k].grad.float()))


def _dgrad_model(dtype, kin=(7, 7, 7)):
    m = VideoTokenizer(image_size=32, init_dim=64, codebook_size=1024, layers=("residual", "compress_time"),
                       input_conv_kernel_size=kin, use_gan=False, perceptual_loss_weight=0.)
    return m.cuda().to(dtype)


def test_video_gradient_runs_on_the_engine_kernels():
    """A bf16 encode with the video requiring grad at init_dim = 64: the video's gradient is one narrow-tile slab launch per
    conv (conv_log), and the runner counts it as its own data gradient."""
    _require_cuda()
    m = _dgrad_model(torch.bfloat16)
    m.eval()
    v = torch.randn(2, 3, 5, 32, 32, device="cuda", requires_grad=True)
    eng = m.engine
    out = m.encode(v)
    eng.conv_log = []
    (out.float() ** 2).sum().backward()
    torch.cuda.synchronize()
    assert v.grad is not None and v.grad.shape == v.shape and torch.isfinite(v.grad).all()
    recs = [r for r in eng.conv_log if r["Co"] == 3 and r["k"] == (7, 7, 7)]
    assert len(recs) == 1 and recs[0]["kind"] == "slab", eng.conv_log
    eng.conv_log = None


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("graphs", [False, True])
def test_no_grad_calls_unchanged(dtype, graphs):
    """Eval-mode calls on plain inputs and calls under no_grad return tensors without grad_fn, equal bit for bit to the
    no-grad engine path, with CUDA graphs on and off."""
    _require_cuda()
    g = load_golden("mini_io_grad")
    m = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    m.cuda_graphs = graphs
    video = golden_video(g).cuda().to(dtype)
    codes = g["codes"].long().cuda()
    eng = m.engine
    with torch.no_grad():
        want_enc = eng.to_channels_first(eng.encode_cl(video))
        z = want_enc.clone()
        want_dec = eng.decode_cl(eng.to_channels_last(z), True)
        want_codes = eng.decode_cl(eng.codes_to_quantized_cl(codes), True)
    for ctx in (torch.enable_grad, torch.no_grad):
        for _ in range(3):                       # warm-up, capture, replay
            with ctx():
                outs = (m.encode(video), m.decode(z), m.decode_from_code_indices(codes))
            for o, w in zip(outs, (want_enc, want_dec, want_codes)):
                assert o.grad_fn is None and not o.requires_grad
                assert torch.equal(o, w)
    m.train()
    with torch.no_grad():
        o = m.decode(z)
    assert o.grad_fn is None


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_train_mode_values_equal_the_no_grad_call(dtype):
    """A train-mode differentiable decode computes the no-grad train-mode call's values: bit for bit in fp32, allclose in
    bf16 (the differentiable path runs the ResidualUnit unfused)."""
    _require_cuda()
    g = load_golden("mini_io_grad")
    m = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    m.train()
    z = _latents(m, g["codes"]).cuda().to(dtype)
    with torch.no_grad():
        want = m.decode(z)
    got = m.decode(z)
    assert got.grad_fn is not None
    if dtype == torch.float32:
        assert torch.equal(got.detach(), want)
    else:
        torch.testing.assert_close(got.detach().float(), want.float(), rtol=3e-2, atol=3e-2)


def test_single_backward():
    _require_cuda()
    g = load_golden("mini_io_grad")
    m = build_product(g["kwargs"], g["wseed"]).cuda()
    z = _latents(m, g["codes"]).cuda().requires_grad_(True)
    loss = m.decode(z).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="backward ran already"):
        loss.backward()


def test_eval_lfq_quantize_with_frozen_quantiser():
    """Eval mode, LFQ, quantize=True, a video requiring grad and every parameter frozen: the quantised value is a constant
    of the video, so a loss that contains it backpropagates to nothing, as in the reference."""
    _require_cuda()
    g = load_golden("mini_io_grad")
    m = build_product(g["kwargs"], g["wseed"]).cuda()
    m.requires_grad_(False)
    v = golden_video(g).cuda().requires_grad_(True)
    q = m.encode(v, quantize=True)[0]
    other = (v ** 2).sum()
    (q.sum() + other).backward()
    torch.testing.assert_close(v.grad, 2 * v.detach())
    assert all(p.grad is None for p in m.parameters())
