"""The perceptual (VGG) loss and the adaptive adversarial weight on the device (vgg.py, train.py, gan.py): the ReLU
epilogue and the 2x2 max-pool kernels against float64, the VGG and the seeded generator step against the unmodified
reference (tests/golden/mini_vgg16.pt, mini_vgg_narrow.pt, oracle/make_vgg_golden.py)."""
import pytest
import torch
import torch.nn.functional as F

import synth_data
from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200 import vgg as V
from magvit2_pytorch_b200._lib import ACT_RELU
from magvit2_pytorch_b200.engine import Engine, PackCache, pack_conv
from tests.test_oracle import grad_digest_close
from tests.util import golden_video, load_golden

pytestmark = pytest.mark.gpu
GOLDENS = ["mini_vgg16", "mini_vgg_narrow"]


@pytest.fixture(autouse=True)
def _no_tf32():
    """cuDNN (the tokenizer's weight gradients) in true fp32; restored even when a test fails."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _engine(dtype):
    eng = Engine(None)
    eng.dtype, eng.device = dtype, torch.device("cuda")
    return eng


def _vgg(g):
    s = g["vgg"]
    return synth_data.fill_vgg_(synth_data.build_vgg(s["cfg"], s["hidden"], s["num_classes"]), g["vseed_vgg"])


def _model(g, dtype=torch.float32):
    torch.manual_seed(0)
    m = VideoTokenizer(**g["kwargs"], vgg=_vgg(g))
    synth_data.fill_state_dict_(m, g["wseed"])
    synth_data.fill_discr_(m, g["wseed"])
    return m.cuda().to(dtype)


def _images(g, dtype=torch.float32):
    return torch.randn(2, 3, 32, 32, generator=torch.Generator(device="cpu").manual_seed(g["iseed"])).to(dtype).cuda()


# ---- kernels against float64
RELU_CASES = [
    # name, (Co, Ci, kh, kw), (B, H, W), dtype, tc_variant: odd / non-tile-multiple maps exercise the tile and padding edges
    ("simt_fp32", (24, 5, 3, 3), (2, 7, 9), torch.float32, None),
    ("slab_bf16", (64, 64, 3, 3), (2, 13, 11), torch.bfloat16, "auto"),
    ("tap_bf16", (96, 32, 3, 3), (2, 9, 15), torch.bfloat16, "tap"),
]


@pytest.mark.parametrize("case", RELU_CASES, ids=[c[0] for c in RELU_CASES])
def test_relu_epilogue_matches_float64(case):
    name, wshape, (B, H, W), dt, variant = case
    gen = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    w = torch.randn(wshape, generator=gen) * (wshape[1] * 9) ** -0.5
    b = torch.randn(wshape[0], generator=gen) * 0.3
    x = torch.randn(B, 1, H, W, wshape[1], generator=gen).to(dt)
    eng = _engine(dt)
    if variant:
        eng.tc_variant = variant
    y = eng.conv(x.cuda(), pack_conv(w.cuda(), b.cuda(), dt), act=ACT_RELU)
    if dt == torch.bfloat16:
        assert eng.tc_calls == 1, "wgmma path was not taken"
    ref = F.relu(F.conv2d(x[:, 0].permute(0, 3, 1, 2).double(), w.to(dt).double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    err = (y[:, 0].double().cpu() - ref).abs().max().item()
    tol = 1e-5 if dt == torch.float32 else 2e-2 * ref.abs().max().item()
    assert err <= tol, (name, err)
    assert (y.float() >= 0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(3, 8, 8, 64), (2, 7, 9, 12), (1, 5, 6, 3)], ids=["vec", "odd_c12", "odd_c3"])
def test_maxpool_forward_backward_match_float64(dtype, shape):
    N, H, W, C = shape
    gen = torch.Generator(device="cpu").manual_seed(N * 100 + C)
    x = F.relu(torch.randn(N, H, W, C, generator=gen)).to(dtype)
    x[0, 0:2, 0:2, 0] = 0.75                      # an all-equal positive window: the gradient goes to its first element
    x[0, 2:4, 2:4, 1] = 0.                        # an all-zero window: the ReLU mask stops its gradient
    eng = _engine(dtype)
    xc = x.cuda()[:, None]
    y = eng.maxpool2x2(xc)
    xr = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.max_pool2d(xr, 2, 2)
    assert torch.equal(y[:, 0].double().cpu(), yr.detach().permute(0, 2, 3, 1))
    g = torch.randn(yr.shape, generator=gen).to(dtype).double()
    gx_ref, = torch.autograd.grad(yr, xr, g)
    gx_ref = gx_ref * (xr.detach() > 0)           # the ReLU before the pool
    gx = eng.maxpool2x2_backward(g.permute(0, 2, 3, 1).to(dtype).cuda()[:, None], xc)
    assert torch.equal(gx[:, 0].double().cpu(), gx_ref.permute(0, 2, 3, 1))
    assert gx[0, 0, 0, 0, 0].item() == g[0, 0, 0, 0].to(dtype).item() and not gx[0, 0, 0:2, 0:2, 0].flatten()[1:].any()


# ---- the VGG and the generator step against the reference
@pytest.mark.parametrize("name", GOLDENS)
def test_fp32_features_vs_reference(name):
    g = load_golden(name)
    vgg = _vgg(g).cuda().eval()
    x = _images(g)
    r = V.VggRunner(vgg, (32, 32))
    feats = r.forward(x)
    ref = g["standalone"]["features"]
    assert ((feats.cpu() - ref).abs().max() / ref.abs().max()).item() < 1e-5
    gx = r.backward(torch.ones_like(feats))
    grad_digest_close(gx, g["standalone"]["grad_images"], 5e-3, "images")


def _gen_step(m, g, video):
    for _, p in m.named_parameters():
        p.grad = None
    torch.manual_seed(g["step_seed"])
    return m(video, return_loss=True)


@pytest.mark.parametrize("name", GOLDENS)
def test_fp32_generator_step_vs_reference(name):
    g = load_golden(name)
    gs = g["gen"]
    m = _model(g)
    m.train()
    m.vgg.eval()
    video = golden_video(g).cuda()
    total, bd = _gen_step(m, g, video)
    for got, key in ((total, "total"), (bd.recon_loss, "recon"), (bd.lfq_aux_loss, "aux"), (bd.perceptual_loss, "perceptual"),
                     (bd.adversarial_gen_loss, "gen")):
        assert abs(float(got) - gs[key].item()) < 1e-5 * max(1., abs(gs[key].item())), (key, float(got), gs[key].item())
    assert torch.is_tensor(bd.adaptive_adversarial_weight)
    assert abs(float(bd.adaptive_adversarial_weight) / gs["adaptive"].item() - 1) < 1e-4, (float(bd.adaptive_adversarial_weight), gs["adaptive"])
    total.backward()
    named = dict(m.named_parameters())
    gnorm = sum(d["norm"] ** 2 for d in gs["grads"].values() if d is not None) ** 0.5
    worst = 0.
    for k, dg in gs["grads"].items():
        p = named[k]
        if dg is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        assert p.grad is not None, k
        worst = max(worst, grad_digest_close(p.grad, dg, 5e-3, k, atol=1e-7 * gnorm))
    # the one difference from the reference: the frozen VGG's parameters get no gradient (no optimizer sees them)
    assert all(p.grad is None for p in m.vgg.parameters())
    print(f"{name}: {len(gs['grads'])} gradients, worst relative deviation {worst:.2e}")
    m.eval()
    torch.manual_seed(g["step_seed"])
    with torch.no_grad():
        total, bd = m(video, return_loss=True)
    ev = g["gen"]["eval"]
    assert bd.adaptive_adversarial_weight == 1.
    for got, key in ((total, "total"), (bd.perceptual_loss, "perceptual"), (bd.adversarial_gen_loss, "gen")):
        assert abs(float(got) - ev[key].item()) < 1e-5 * max(1., abs(ev[key].item())), (key, float(got), ev[key].item())


def test_train_mode_without_gradients_raises():
    g = load_golden("mini_vgg_narrow")
    m = _model(g).train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="gradients"):
        m(golden_video(g).cuda(), return_loss=True)


def test_vgg_without_gan_has_perceptual_term_only():
    g = load_golden("mini_vgg_narrow")
    torch.manual_seed(0)
    m = VideoTokenizer(**dict(g["kwargs"], use_gan=False), vgg=_vgg(g))
    synth_data.fill_state_dict_(m, g["wseed"])
    m = m.cuda().train()
    m.vgg.eval()
    total, bd = _gen_step(m, g, golden_video(g).cuda())
    assert bd.adaptive_adversarial_weight == 0. and float(bd.adversarial_gen_loss) == 0.
    assert abs(float(bd.perceptual_loss) - g["gen"]["perceptual"].item()) < 1e-5 * max(1., g["gen"]["perceptual"].item())
    total.backward()
    assert m.conv_out.conv.weight.grad is not None


@pytest.mark.parametrize("name", GOLDENS)
def test_bf16_within_reference_bf16_error_budget(name):
    g = load_golden(name)
    g16 = g["bf16"]
    m = _model(g, torch.bfloat16)
    m.vgg.eval()
    with torch.no_grad():
        feats = V.VggRunner(m.vgg, (32, 32)).forward(_images(g, torch.bfloat16), record=False).float().cpu()
    pairs = [(feats, g16["standalone"]["features"], g["standalone"]["features"])]
    m.train()
    m.vgg.eval()
    total, bd = _gen_step(m, g, golden_video(g).cuda().bfloat16())
    for got, key in ((total, "total"), (bd.perceptual_loss, "perceptual"), (bd.adversarial_gen_loss, "gen")):
        pairs.append((torch.as_tensor(float(got)), g16["gen"][key], g["gen"][key]))
    # as test_gan_gpu: the standalone features isolate the VGG (1.5x mean / 2x max of the reference's own bf16 error); the
    # step's scalars also carry the bf16 tokenizer's reconstruction, held to 3x.  The perceptual term of the narrow VGG is the
    # exception: it compares the features of the bf16 reconstruction, whose roundings differ from the reference's, and its
    # narrow layers amplify that -- measured on an H100 80GB HBM3 (700 W) at 5.0x the reference's own bf16 error (VGG16
    # layout: 1.4x), held here to 6x
    for i, (got, ref16, ref32) in enumerate(pairs):
        got, ref16, ref32 = got.reshape(-1), ref16.reshape(-1), ref32.reshape(-1)
        e_prod, e_ref = (got - ref32).abs(), (ref16 - ref32).abs()
        print(f"{name} pair {i}: product err mean {e_prod.mean().item():.3e} max {e_prod.max().item():.3e}; reference bf16 err "
              f"mean {e_ref.mean().item():.3e} max {e_ref.max().item():.3e}")
        k_mean, k_max = (1.5, 2.0) if i == 0 else (6.0, 6.0) if (name, i) == ("mini_vgg_narrow", 2) else (3.0, 3.0)
        scale = 1e-3 * max(1., ref32.abs().max().item())
        assert e_prod.mean().item() <= k_mean * e_ref.mean().item() + scale, (i, e_prod, e_ref)
        assert e_prod.max().item() <= k_max * e_ref.max().item() + scale, (i, e_prod, e_ref)
    total.backward()
    assert torch.isfinite(m.conv_out.conv.weight.grad.float()).all()


def test_bf16_vgg_convs_run_on_tensor_cores():
    g = load_golden("mini_vgg16")
    vgg = _vgg(g).cuda().bfloat16().eval()
    cache = PackCache()
    V.VggRunner(vgg, (32, 32), cache=cache).forward(_images(g, torch.bfloat16), record=False)       # packs
    eng = cache.engine
    eng.conv_log, eng.simt_conv_calls = [], 0
    r = V.VggRunner(vgg, (32, 32), cache=cache)
    feats = r.forward(_images(g, torch.bfloat16))
    r.backward(torch.ones_like(feats))
    log, eng.conv_log = eng.conv_log, None
    assert eng.simt_conv_calls == 0, eng.simt_conv_calls
    n_conv = sum(isinstance(mod, torch.nn.Conv2d) for mod in vgg.features)
    assert sum(r_["act"] == ACT_RELU for r_ in log) >= n_conv
    assert any(r_["Ci"] == 32 and r_["k"] == (1, 3, 1) for r_ in log)          # the kw-packed first conv


def test_dropout_masks_follow_vgg_training_and_the_seed():
    g = load_golden("mini_vgg_narrow")
    vgg = _vgg(g).cuda().train()
    real, fake = _images(g), _images(g).flip(0)
    torch.manual_seed(5)
    a, info = V.perceptual_loss(vgg, real, fake)
    masks_real, masks_fake = info["masks"]
    assert sum(m is not None for m in masks_fake) == 2
    with torch.no_grad():
        ref = F.mse_loss(V.vgg_torch(vgg, real, [None if m is None else m.reshape(2, -1) for m in masks_real]),
                         V.vgg_torch(vgg, fake, [None if m is None else m.reshape(2, -1) for m in masks_fake]))
    assert abs(a.item() - ref.item()) <= 1e-5 * abs(ref.item()), (a.item(), ref.item())
    torch.manual_seed(5)
    b, _ = V.perceptual_loss(vgg, real, fake)
    assert a.item() == b.item()


def test_trainer_shaped_loop_bf16():
    g = load_golden("mini_vgg_narrow")
    m = _model(g, torch.bfloat16)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    dopt = torch.optim.AdamW(m.discr_parameters(), lr=1e-4)
    g0 = [p.detach().clone() for p in m.parameters()]
    video = golden_video(g).cuda().bfloat16()
    m.train()
    for step in range(3):
        opt.zero_grad()
        loss, bd = m(video, return_loss=True)
        loss.backward()
        opt.step()
        dopt.zero_grad()
        dloss, _ = m(video, return_discr_loss=True, apply_gradient_penalty=step == 0)
        dloss.backward()
        dopt.step()
        for v in (loss, bd.perceptual_loss, bd.adversarial_gen_loss, bd.adaptive_adversarial_weight, dloss):
            assert torch.isfinite(torch.as_tensor(v).float()).all(), step
    assert any(not torch.equal(a, p) for a, p in zip(g0, m.parameters()))


# ---- the adaptive weight's last-layer gradient, the 1- / 4-channel device path, and the runners' lifetime
LAST_LAYER_CASES = {
    "constant": dict(),
    "replicate": dict(pad_mode="replicate"),
    "sff_reflect": dict(separate_first_frame_encoding=True, pad_mode="reflect"),
}


@pytest.mark.parametrize("case", list(LAST_LAYER_CASES))
def test_last_layer_weight_grad_matches_autograd(case):
    """TrainRunner.last_layer_weight_grad == autograd's conv_out weight gradient for the same reconstruction gradient, with
    time_padding frames (compress_time), the pad modes and separate_first_frame_encoding; the tape stays usable."""
    from magvit2_pytorch_b200.train import TrainRunner, train_forward
    torch.manual_seed(0)
    m = VideoTokenizer(image_size=16, init_dim=16, codebook_size=256, layers=("residual", "compress_time"), use_gan=False,
                       perceptual_loss_weight=0., **LAST_LAYER_CASES[case])
    synth_data.fill_state_dict_(m, 3)
    m = m.cuda().train()
    assert m.time_padding == 1
    gen = torch.Generator(device="cpu").manual_seed(9)
    video = torch.randn(2, 3, 5, 16, 16, generator=gen).cuda()
    runner = TrainRunner(m)
    recon, _, _, _ = train_forward(m, video, runner=runner)
    g = torch.randn(recon.shape, generator=gen).cuda()
    g[:, :, 0] *= 3.                                  # the first frame (conv_out_first_frame under sff) weighs differently
    gw = runner.last_layer_weight_grad(g)
    w = m.conv_out.conv.weight
    ref, = torch.autograd.grad(recon, w, g)
    err = ((gw - ref).abs().max() / ref.abs().max()).item()
    assert err < 1e-5, (case, err)
    with pytest.raises(RuntimeError, match="released"):
        runner.last_layer_weight_grad(g)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("channels", [1, 4])
def test_one_and_four_channel_frames_match_reference_repeat_and_slice(channels, dtype):
    """channels 1 / 4 (M:1797-1803) on the device: the folded first conv (kw-packed ingest in bf16) and its data gradient
    back to the frames' own channels, against float64 autograd through the reference's repeat / slice."""
    import copy
    vgg = synth_data.fill_vgg_(synth_data.build_vgg((16, "M", 32, "M", 64, 64, "M"), 64, num_classes=32), 4).eval()
    vgg64 = copy.deepcopy(vgg).to(dtype).double()
    vgg = vgg.cuda().to(dtype)
    gen = torch.Generator(device="cpu").manual_seed(channels)
    x = torch.randn(2, channels, 32, 32, generator=gen).to(dtype)
    gf = torch.randn(2, 32, generator=gen).to(dtype)
    cache = PackCache()
    r = V.VggRunner(vgg, (32, 32), channels, cache)
    feats = r.forward(x.cuda())
    gx = r.backward(gf.cuda())
    if dtype == torch.bfloat16:
        assert "kw" in cache.packs["feats"][0]
    xr = x.double().requires_grad_(True)
    ref = V.vgg_torch(vgg64, xr.repeat(1, 3, 1, 1) if channels == 1 else xr[:, :3])
    gref, = torch.autograd.grad(ref, xr, gf.double())
    tol = 1e-4 if dtype == torch.float32 else 4e-2
    assert ((feats.double().cpu() - ref.detach()).abs().max() / ref.abs().max()).item() < tol
    gx64 = gx.double().cpu()
    if dtype == torch.float32:
        assert ((gx64 - gref).abs().max() / gref.abs().max()).item() < tol
    else:
        # in bf16 a ReLU mask or a pool's argmax that flips under rounding moves a whole gradient entry: the data gradient is
        # held, in norm, to 2x the error of torch's own bf16 autograd through the reference's repeat / slice
        xt = x.cuda().requires_grad_(True)
        ft = V.vgg_torch(vgg, xt.repeat(1, 3, 1, 1) if channels == 1 else xt[:, :3])
        gt, = torch.autograd.grad(ft, xt, gf.cuda())
        rel = ((gx64 - gref).norm() / gref.norm()).item()
        rel_torch = ((gt.double().cpu() - gref).norm() / gref.norm()).item()
        print(f"channels {channels} bf16: data gradient relative L2 error {rel:.3e}, torch bf16 {rel_torch:.3e}")
        assert rel <= 2 * rel_torch + 1e-3, (rel, rel_torch)
    assert gx.shape == x.shape
    if channels == 4:
        assert not gx[:, 3].any()                    # the dropped 4th channel gets no gradient


def test_runners_are_freed_with_the_loss_graph(monkeypatch):
    """No runner of a VGG + GAN generator step outlives `loss.backward(); del loss`: their saved activations and gradient
    dicts are freed by reference counting, without a cyclic collection."""
    import gc
    import weakref
    from magvit2_pytorch_b200 import gan as G
    from magvit2_pytorch_b200 import train as T
    refs = []

    def tracked(cls):
        class Tracked(cls):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                refs.append(weakref.ref(self))
        return Tracked

    monkeypatch.setattr(T, "TrainRunner", tracked(T.TrainRunner))
    monkeypatch.setattr(G, "DiscrRunner", tracked(G.DiscrRunner))
    monkeypatch.setattr(V, "VggRunner", tracked(V.VggRunner))
    g = load_golden("mini_vgg_narrow")
    m = _model(g).train()
    video = golden_video(g).cuda()
    gc.collect()
    gc.disable()
    try:
        loss, bd = m(video, return_loss=True)
        loss.backward()
        del loss, bd
        alive = [type(r()).__mro__[1].__name__ for r in refs if r() is not None]
    finally:
        gc.enable()
    assert len(refs) == 4, len(refs)                  # tokenizer, VGG on real and recon frames, discriminator
    assert not alive, alive
