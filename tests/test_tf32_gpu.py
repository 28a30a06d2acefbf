"""fp32 tokenizers with torch's TF32 matmul switch on: the no-grad calls run their dense contractions on the TF32 tensor
cores, on the fp32 fixtures (mini, readme, fsq, mini_gateloop):

  * codes: every bit whose sign differs from the fixture's has an fp32 pre-sign value below TAU (LFQ fixtures);
  * accuracy: the decode of the fixture's codes is no further from the reference than the product's own bf16 decode;
  * two runs agree bit for bit; CUDA graphs, lanes, HostRoundTrip and streams give the eager TF32 outputs bit for bit;
  * switching TF32 off restores the IEEE outputs bit for bit; a call with gradients launches no tensor-core conv with the
    switch on and its forward gives the same bits either way (the pieces of its backward that torch runs, such as cuDNN
    weight gradients, follow torch's own switches, as in the reference).
The `tf32` fixture restores torch's switch however a test ends."""
import pytest
import torch

from magvit2_pytorch_b200 import HostRoundTrip, StreamLanes
from tests.util import build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu

# |fp32 pre-sign value| below which a token may flip: TF32 reads operands with 10 mantissa bits (relative error 2^-10 per
# operand), and the pre-sign values of the fixtures are O(1)
TAU = 2e-2
NAMES = ["mini", "readme", "fsq", "mini_gateloop"]


@pytest.fixture
def tf32():
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev


def _model(g, dtype=torch.float32):
    return build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)


def _recon_err(recon, g):
    if "recon" in g:
        return (recon.float().cpu() - g["recon"]).abs()
    return (recon.float().cpu()[:, :, :, ::4, ::4] - g["recon_sample"]).abs()


@pytest.mark.parametrize("name", NAMES)
def test_tf32_codes_and_decode_vs_fixture(tf32, name):
    g = load_golden(name)
    model = _model(g)
    video = golden_video(g).cuda()
    eng = model.engine
    tc0 = eng.tc_calls
    codes = model.tokenize(video)
    assert eng.tc_calls > tc0, "TF32 did not run on the tensor cores"
    assert eng.simt_conv_calls == 0, "a TF32 conv ran on the CUDA cores"
    lfq = not g["kwargs"].get("use_fsq", False)
    if lfq:
        # the pre-sign values of the same TF32 encode: every bit whose sign differs from the fixture's is near zero there
        eng = model._tf32_engine()
        try:
            _, codes_e, pre = eng.quantize_cl(eng.encode_cl(video), want_quantized=False, want_aux=True)
        finally:
            eng.tf32 = False
        assert torch.equal(codes_e.reshape(codes.shape), codes)
        p32 = g["presign"]
        flipped = (pre.cpu().reshape(p32.shape) > 0) != (p32 > 0)
        if flipped.any():
            assert p32[flipped].abs().max().item() < TAU, p32[flipped].abs().max().item()
        assert torch.equal((codes.cpu() != g["codes"]).any(), flipped.any())
    else:
        assert (codes.cpu() != g["codes"]).float().mean().item() <= 0.02
    recon = model.decode_from_code_indices(g["codes"].cuda())
    assert recon.dtype == torch.float32
    m16 = _model(g, torch.bfloat16)
    r16 = m16.decode_from_code_indices(g["codes"].cuda())
    e32, e16 = _recon_err(recon, g), _recon_err(r16, g)
    assert e32.max().item() <= e16.max().item() and e32.mean().item() <= e16.mean().item(), (e32.max(), e16.max())


@pytest.fixture(scope="module")
def readme():
    g = load_golden("readme")
    return g, golden_video(g).cuda()


def _run(model, video):
    codes = model.tokenize(video)
    return codes, model.decode_from_code_indices(codes)


def test_tf32_deterministic_and_switch_off_restores_ieee(readme):
    g, video = readme
    model = _model(g)
    c_ieee, r_ieee = _run(model, video)
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        tc0 = model.engine.tc_calls
        c1, r1 = _run(model, video)
        c2, r2 = _run(model, video)
        assert model.engine.tc_calls > tc0
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    assert torch.equal(c1, c2) and torch.equal(r1, r2)
    assert not torch.equal(r1, r_ieee)
    tc0 = model.engine.tc_calls
    c3, r3 = _run(model, video)
    assert model.engine.tc_calls == tc0
    assert torch.equal(c3, c_ieee) and torch.equal(r3, r_ieee)


def test_tf32_replay_modes_match_eager(tf32, readme):
    g, video = readme
    model = _model(g)
    codes, recon = _run(model, video)
    model.cuda_graphs = True
    for _ in range(3):
        c, r = _run(model, video)
        assert torch.equal(c, codes) and torch.equal(r, recon)
    lanes = StreamLanes(model, 2)
    outs = [lanes.run(_run, model, video)[0] for _ in range(3)]
    lanes.join()
    for c, r in outs:
        assert torch.equal(c, codes) and torch.equal(r, recon)
    model.cuda_graphs = False
    hrt = HostRoundTrip(model, depth=2)
    vh = video.cpu().pin_memory()
    ch, rh = torch.empty(codes.shape, dtype=codes.dtype).pin_memory(), torch.empty(recon.shape).pin_memory()
    hrt.wait(hrt.submit(vh, ch, rh))
    assert torch.equal(ch, codes.cpu()) and torch.equal(rh, recon.cpu())
    # streams: chunks of the clip give the whole-clip codes; latent chunks give the whole-clip frames
    tdf = model.time_downsample_factor
    ts = model.tokenize_stream(video.shape[0])
    sc = torch.cat([ts.push(video[:, :, :1 + tdf]), ts.push(video[:, :, 1 + tdf:])], 1)
    assert torch.equal(sc, codes)
    ds = model.decode_stream(video.shape[0])
    sr = torch.cat([ds.push(codes[:, :2]), ds.push(codes[:, 2:])], 2)
    assert torch.equal(sr, recon)


def test_stream_keeps_its_precision(readme):
    g, video = readme
    model = _model(g)
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        codes = model.tokenize(video)
        ts = model.tokenize_stream(video.shape[0])
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    tdf = model.time_downsample_factor
    sc = torch.cat([ts.push(video[:, :, :1 + tdf]), ts.push(video[:, :, 1 + tdf:])], 1)   # switch off by now
    assert torch.equal(sc, codes)


def test_gradient_calls_ignore_the_switch(tf32):
    g = load_golden("mini")
    model = _model(g)
    video = golden_video(g).cuda()
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    z0 = model.encode(video.clone().requires_grad_(True)).detach()
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    tc0 = model.engine.tc_calls
    v = video.clone().requires_grad_(True)
    z1 = model.encode(v)
    z1.square().sum().backward()
    assert model.engine.tc_calls == tc0 and v.grad is not None
    assert torch.equal(z0, z1.detach())
    assert not torch.equal(model.encode(video), z0)          # the same call without gradients follows the switch


def test_no_grad_losses_follow_the_switch(readme):
    """eval return_recon_loss_only and lfq_loss_breakdown run TF32 with the switch on, and give the IEEE bits again with it
    off (the README model's loss has a perceptual term, so its return_loss needs a VGG)."""
    g, video = readme
    model = _model(g)

    def calls():
        rl, _ = model(video, return_recon_loss_only=True)
        codes, (ps, be, cm), aux = model.lfq_loss_breakdown(video)
        return torch.stack([rl, ps, be, cm, aux]), codes

    v_ieee, c_ieee = calls()
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        tc0 = model.engine.tc_calls
        v_tf32, _ = calls()
        assert model.engine.tc_calls > tc0
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    assert not torch.equal(v_tf32, v_ieee)
    # the entropy terms average soft code probabilities over 1280 tokens: a few 1e-3 apart in TF32
    assert torch.allclose(v_tf32, v_ieee, rtol=2e-2, atol=5e-3), (v_tf32, v_ieee)
    v2, c2 = calls()
    # the reconstruction loss and the codes give the IEEE bits again (the entropy terms reduce in no fixed order)
    assert torch.equal(v2[0], v_ieee[0]) and torch.equal(c2, c_ieee)
    assert torch.allclose(v2, v_ieee, rtol=1e-5, atol=1e-7)


def test_discriminator_ignores_the_switch():
    """return_discr_loss and an eval return_loss with the image discriminator: the same bits with the switch on and off
    (the discriminator runs on an engine of its own, and the tokenizer forward of these calls stays IEEE)."""
    import synth_data
    from magvit2_pytorch_b200 import VideoTokenizer
    g = load_golden("mini_gan")
    torch.manual_seed(0)
    m = VideoTokenizer(**g["kwargs"])
    synth_data.fill_state_dict_(m, g["wseed"])
    synth_data.fill_discr_(m, g["wseed"])
    m = m.cuda().eval()
    video = golden_video(g).cuda()

    def calls():
        torch.manual_seed(1)
        d, _ = m(video, return_discr_loss=True, apply_gradient_penalty=False)
        torch.manual_seed(2)
        with torch.no_grad():
            t, _ = m(video, return_loss=True)
        return torch.stack([d.detach(), t])

    off = calls()
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        tc0 = m.engine.tc_calls
        on = calls()
        assert m.engine.tc_calls == tc0
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    assert torch.equal(on, off), (on, off)


def test_causal_conv_transpose_follows_the_switch():
    """The standalone CausalConvTranspose3d: TF32 on the tensor cores with the switch on, its IEEE bits with it off, and one
    pack for both (toggling the switch re-packs nothing)."""
    from magvit2_pytorch_b200.modules import CausalConvTranspose3d
    torch.manual_seed(0)
    mod = CausalConvTranspose3d(64, 32, 3, time_stride=2).cuda()
    x = torch.randn(2, 64, 3, 8, 8, device="cuda")
    with torch.no_grad():
        y_ieee = mod(x)
        packs = mod._pack_cache.packs
        eng = mod._pack_cache.engine
        prev = torch.backends.cuda.matmul.fp32_precision
        torch.backends.cuda.matmul.fp32_precision = "tf32"
        try:
            tc0 = eng.tc_calls
            y_tf32 = mod(x)
            assert eng.tc_calls == tc0 + 1
        finally:
            torch.backends.cuda.matmul.fp32_precision = prev
        y2 = mod(x)
    assert mod._pack_cache.packs is packs
    assert torch.equal(y2, y_ieee) and not torch.equal(y_tf32, y_ieee)
    assert (y_tf32 - y_ieee).abs().max().item() <= 1e-2 * y_ieee.abs().max().item()
