"""The GAN discriminator on the device (gan.py) against the unmodified reference (tests/golden/mini_gan.pt,
mini_gan_bf16.pt, oracle/make_gan_golden.py), and its new tensor-core conv flavours against the CUDA-core conv."""
import pytest
import torch
import torch.nn.functional as F

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200 import gan
from magvit2_pytorch_b200._lib import ACT_LEAKY_RELU, ACT_NONE, SHUFFLE_SPACE
from magvit2_pytorch_b200.engine import Engine, pack_conv
from tests.test_oracle import grad_digest_close
from tests.util import golden_video, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_tf32():
    """cuDNN (the weight gradients, the penalty's restatement) in true fp32; restored even when a test fails."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _model(g, dtype=torch.float32):
    torch.manual_seed(0)
    m = VideoTokenizer(**g["kwargs"])
    synth_data.fill_state_dict_(m, g["wseed"])
    synth_data.fill_discr_(m, g["wseed"])
    return m.cuda().to(dtype)


def _images(g, dtype=torch.float32):
    gen = torch.Generator(device="cpu").manual_seed(g["iseed"])
    return torch.randn(2, 3, 32, 32, generator=gen).to(dtype).cuda()


def _zero(m):
    for _, p in m.named_parameters():
        p.grad = None


def _check_grads(named, digests, what):
    gnorm = sum(d["norm"] ** 2 for d in digests.values() if d is not None) ** 0.5
    worst = 0.0
    for k, dg in digests.items():
        if k not in named:
            continue
        p = named[k]
        if dg is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, (what, k)
            continue
        assert p.grad is not None, (what, k)
        worst = max(worst, grad_digest_close(p.grad, dg, 5e-3, f"{what}:{k}", atol=1e-7 * gnorm))
    return worst


def test_fp32_standalone_vs_reference():
    g = load_golden("mini_gan")
    m = _model(g)
    x = _images(g).requires_grad_(True)
    logits = m.discr(x)
    assert logits.shape == (2,) and logits.dtype == torch.float32
    ref = g["standalone"]["logits"]
    assert ((logits.detach().cpu() - ref).abs() / ref.abs()).max().item() < 1e-5
    logits.sum().backward()
    grad_digest_close(x.grad, g["standalone"]["grad_images"], 5e-3, "images")
    _check_grads(dict(m.discr.named_parameters()), g["standalone"]["grads"], "standalone")
    with pytest.raises(RuntimeError):             # first-order only, as once_differentiable
        y = _images(g).requires_grad_(True)
        gx, = torch.autograd.grad(m.discr(y).sum(), y, create_graph=True)
        gx.sum().backward()


@pytest.mark.parametrize("step", ["discr", "discr_gp", "gen"])
def test_fp32_steps_vs_reference(step):
    g = load_golden("mini_gan")
    gs = g[step]
    m = _model(g)
    m.train()
    _zero(m)
    torch.manual_seed(g["step_seed"])
    video = golden_video(g).cuda()
    if step == "gen":
        total, bd = m(video, return_loss=True)
        assert abs(bd.recon_loss.item() - gs["recon"].item()) < 1e-5
        assert abs(bd.adversarial_gen_loss.item() - gs["gen"].item()) < 1e-5
        assert bd.adaptive_adversarial_weight == 1.
        named = dict(m.named_parameters())
    else:
        total, bd = m(video, return_discr_loss=True, apply_gradient_penalty=step == "discr_gp")
        assert abs(bd.discr_loss.item() - gs["hinge"].item()) < 1e-5
        assert abs(float(bd.gradient_penalty.detach()) - gs["penalty"].item()) < 1e-5
        assert len(bd.multiscale_discr_losses) == 1
        named = {"discr." + k: p for k, p in m.discr.named_parameters()}
    assert abs(total.item() - gs["total"].item()) < 1e-5 * max(1., abs(gs["total"].item()))   # penalty steps: 10 x penalty
    total.backward()
    worst = _check_grads(named, gs["grads"], step)
    print(f"{step}: {len(gs['grads'])} gradients, worst relative deviation {worst:.2e}")


def test_bf16_within_reference_bf16_error_budget():
    g32, g16 = load_golden("mini_gan"), load_golden("mini_gan_bf16")
    m = _model(g32, torch.bfloat16)
    with torch.no_grad():
        logits = m.discr(_images(g32, torch.bfloat16)).float().cpu()
    pairs = [(logits, g16["logits"], g32["standalone"]["logits"])]
    m.train()
    video = golden_video(g32).cuda().bfloat16()
    torch.manual_seed(g32["step_seed"])
    total, bd = m(video, return_discr_loss=True, apply_gradient_penalty=False)
    pairs += [(total.float().cpu(), g16["discr"]["total"], g32["discr"]["total"])]
    torch.manual_seed(g32["step_seed"])
    total, bd = m(video, return_loss=True)
    pairs += [(total.detach().float().cpu(), g16["gen"]["total"], g32["gen"]["total"]),
              (bd.adversarial_gen_loss.detach().float().cpu(), g16["gen"]["gen"], g32["gen"]["gen"])]
    # the standalone logits isolate the discriminator: 1.5x (mean) / 2x (max) of the reference's own bf16 error.  The step
    # losses also carry the bf16 tokenizer's reconstruction, whose roundings differ from the reference's, on one frame per
    # clip; measured on the H100 they deviate 2.3-2.5x the reference's own bf16 error on these scalars, held here to 3x
    for i, (got, ref16, ref32) in enumerate(pairs):
        got, ref16, ref32 = got.detach().reshape(-1), ref16.reshape(-1), ref32.reshape(-1)
        e_prod, e_ref = (got - ref32).abs(), (ref16 - ref32).abs()
        print(f"pair {i}: product err {e_prod.tolist()} reference bf16 err {e_ref.tolist()}")
        k_mean, k_max = (1.5, 2.0) if i == 0 else (3.0, 3.0)
        assert e_prod.mean().item() <= k_mean * e_ref.mean().item() + 1e-3, (i, e_prod, e_ref)
        assert e_prod.max().item() <= k_max * e_ref.max().item() + 1e-3, (i, e_prod, e_ref)


def test_bf16_discriminator_convs_run_on_tensor_cores():
    g = load_golden("mini_gan")
    m = _model(g, torch.bfloat16)
    with torch.no_grad():
        m.discr(_images(g, torch.bfloat16))               # packs, engine
        eng = m.discr._pack_cache.engine
        eng.conv_log, eng.simt_conv_calls = [], 0
        m.discr(_images(g, torch.bfloat16))
    log, eng.conv_log = eng.conv_log, None
    # every conv with Ci >= 16 and the kw-packed first conv are wgmma launches; only the 3-channel conv_res stays on the
    # CUDA cores
    assert eng.simt_conv_calls == 1, eng.simt_conv_calls
    assert any(r["Ci"] == 32 and r["k"] == (1, 3, 1) and r["act"] == ACT_LEAKY_RELU for r in log)     # kw-packed first conv
    assert sum(r["epi_mode"] == 2 for r in log) == len(m.discr.blocks)
    assert any(r["stride"] == (1, 2, 2) and r["k"] == (1, 2, 2) for r in log)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_discriminator_is_deterministic(dtype):
    g = load_golden("mini_gan")
    m = _model(g, dtype)
    with torch.no_grad():
        a, b = m.discr(_images(g, dtype)), m.discr(_images(g, dtype))
    assert torch.equal(a, b)


# ---- the new tensor-core flavours against the fp32 CUDA-core conv
def _engine(dtype):
    eng = Engine(None)
    eng.dtype, eng.device = dtype, torch.device("cuda")
    return eng


TC_CASES = [
    # name, weight shape, x shape (B,T,H,W), conv kwargs, epi_mode, variant
    ("leaky_slab", (64, 64, 1, 3, 3), (2, 1, 16, 16), dict(act=ACT_LEAKY_RELU), 0, "auto"),
    ("leaky_tap", (64, 64, 1, 3, 3), (2, 1, 16, 16), dict(act=ACT_LEAKY_RELU), 0, "tap"),
    ("scaled_res_slab", (64, 64, 1, 1, 1), (2, 1, 16, 16), dict(res=True), 2, "auto"),
    ("scaled_res_leaky_tap", (64, 64, 1, 3, 3), (2, 1, 16, 16), dict(res=True, act=ACT_LEAKY_RELU), 2, "tap"),
    ("unshuffle_2x2_s2", (64, 64, 1, 2, 2), (2, 1, 16, 16), dict(res=True, stride=(1, 2, 2), pad=(0, 0, 0)), 2, "auto"),
    ("conv_res_1x1_s2", (128, 64, 1, 1, 1), (2, 1, 16, 16), dict(stride=(1, 2, 2), pad=(0, 0, 0)), 0, "auto"),
    ("dgrad_unshuffle", (256, 64, 1, 1, 1), (2, 1, 8, 8), dict(shuffle=SHUFFLE_SPACE), 0, "auto"),
    ("logits_linear", (1, 64, 1, 4, 4), (2, 1, 4, 4), dict(pad=(0, 0, 0), out_spatial=(1, 1, 1)), 0, "auto"),
]


@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tc_flavours_match_cuda_core(case):
    name, wshape, xshape, kw, epi_mode, variant = case
    kw = dict(kw)
    gen = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    fan_in = wshape[1] * wshape[2] * wshape[3] * wshape[4]
    w = torch.randn(wshape, generator=gen) * fan_in ** -0.5
    bias = torch.randn(wshape[0], generator=gen) * 0.1
    B, T, H, W = xshape
    x = torch.randn((B, T, H, W, wshape[1]), generator=gen).to(torch.bfloat16)
    stride = kw.get("stride", (1, 1, 1))
    if "out_spatial" not in kw:
        kw["out_spatial"] = (T, H // stride[1], W // stride[2])
    co = wshape[0] // 4 if kw.get("shuffle") == SHUFFLE_SPACE else wshape[0]
    osz = kw["out_spatial"] if kw.get("shuffle") != SHUFFLE_SPACE else (T, 2 * H, 2 * W)
    res = torch.randn((B, *osz, co), generator=gen).to(torch.bfloat16) if kw.pop("res", False) else None

    def run(eng, use_tc, dt):
        q = 4 if kw.get("shuffle") == SHUFFLE_SPACE else 1
        pk = pack_conv(w.cuda(), bias.cuda(), dt, shuffle_q=q)
        pk.epi_mode = epi_mode
        eng.use_tc, eng.tc_variant = use_tc, variant
        eng.tc_calls = 0
        y = eng.conv(x.cuda().to(dt), pk, res=None if res is None else res.cuda().to(dt), **kw)
        return y, eng.tc_calls

    y_tc, n_tc = run(_engine(torch.bfloat16), True, torch.bfloat16)
    assert n_tc == 1, "wgmma path was not taken"
    y32, _ = run(_engine(torch.float32), False, torch.float32)
    torch.cuda.synchronize()
    err = (y_tc.float() - y32).abs()
    scale = y32.abs().max().item()
    assert err.max().item() <= 2e-2 * scale + 1e-2, (name, err.max().item(), scale)
    assert err.mean().item() <= 4e-3 * scale, (name, err.mean().item(), scale)


def test_trainer_shaped_loop_bf16():
    """Three iterations of the reference trainer's step (T:339-446): generator step, AdamW, discriminator step (penalty on the
    first), AdamW."""
    g = load_golden("mini_gan")
    m = _model(g, torch.bfloat16)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    dopt = torch.optim.AdamW(m.discr_parameters(), lr=1e-4)
    g0 = [p.detach().clone() for p in m.parameters()]
    d0 = [p.detach().clone() for p in m.discr_parameters()]
    video = golden_video(g).cuda().bfloat16()
    m.train()
    for step in range(3):
        opt.zero_grad()
        loss, bd = m(video, return_loss=True)
        loss.backward()
        opt.step()
        dopt.zero_grad()
        dloss, dbd = m(video, return_discr_loss=True, apply_gradient_penalty=step == 0)
        dloss.backward()
        dopt.step()
        for v in (loss, bd.adversarial_gen_loss, dloss, dbd.discr_loss, dbd.gradient_penalty):
            assert torch.isfinite(torch.as_tensor(v).float()).all(), step
    assert any(not torch.equal(a, p) for a, p in zip(g0, m.parameters()))
    assert any(not torch.equal(a, p) for a, p in zip(d0, m.discr_parameters()))
    m.eval()
    with torch.no_grad():
        _, bd = m(video, return_loss=True)
    assert bd.adaptive_adversarial_weight == 1. and torch.isfinite(bd.adversarial_gen_loss.float())
