"""Pins oracle/restated.py (the CPU restatement used as the checker on the GPU box) against
golden vectors produced by the unmodified reference (oracle/make_golden.py), and checks the
behavioural properties SURVEY.md section 4 lists.  CPU only."""
import pytest
import torch

from tests.util import (build_oracle, build_oracle_from_golden, build_product, golden_video, load_golden,
                        sample_like_golden)

SMALL = ["cfg1", "mini", "mini_fsq", "mini_gateloop", "mini_mc", "mini_mc_fsq"]


@pytest.mark.parametrize("name", SMALL)
def test_restated_matches_reference_golden(name):
    g = load_golden(name)
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    video = golden_video(g)
    taps = {}
    codes = orc.tokenize(video, taps=taps)
    assert codes.dtype == g["codes"].dtype
    assert torch.equal(codes, g["codes"]), "restated oracle codes differ from the reference's"
    for k, ref in g["taps"].items():
        if k.startswith("enc") or k == "conv_in":
            got = sample_like_golden(taps[k], g)
            assert torch.allclose(got, ref, atol=2e-5, rtol=1e-5), k
    dtaps = {}
    recon = orc.decode_from_code_indices(codes, taps=dtaps)
    assert torch.allclose(recon, g["recon"], atol=2e-5, rtol=1e-5)
    for k, ref in g["taps"].items():
        if k.startswith("dec"):
            assert torch.allclose(sample_like_golden(dtaps[k], g), ref, atol=2e-5, rtol=1e-5), k


def test_restated_matches_reference_golden_readme():
    """BASELINE configs[1] (README config), one clip: ~6 s of CPU."""
    g = load_golden("readme")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    video = golden_video(g)
    codes, pre = orc.tokenize(video, return_presign=True)
    assert torch.equal(codes, g["codes"])
    assert torch.allclose(pre, g["presign"], atol=1e-4)
    recon = orc.decode_from_code_indices(codes)
    assert torch.allclose(recon[:, :, :, ::4, ::4], g["recon_sample"], atol=5e-5, rtol=1e-5)
    assert torch.allclose(recon.mean(dim=(3, 4)), g["recon_mean"], atol=1e-5)


def test_restated_matches_reference_golden_fsq_full_size():
    """BASELINE configs[4] (README layers, FSQ [8,5,5,5]) at full size, one clip."""
    g = load_golden("fsq")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    codes = orc.tokenize(golden_video(g))
    assert codes.dtype == torch.int32 and torch.equal(codes, g["codes"])
    recon = orc.decode_from_code_indices(codes)
    assert torch.allclose(recon[:, :, :, ::4, ::4], g["recon_sample"], atol=5e-5, rtol=1e-5)


def test_restated_matches_reference_golden_cfg4_tokenize():
    """BASELINE configs[3] (image 256, max_dim 1024; space-attention seq 1024, linear-attention seq 4096): tokenize side
    (~30 s of CPU; the decode side is pinned on the GPU box through the product, tests/test_parity_gpu.py)."""
    g = load_golden("cfg4")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    taps = {}
    codes, pre = orc.tokenize(golden_video(g), taps=taps, return_presign=True)
    assert torch.equal(codes, g["codes"])
    assert torch.allclose(pre, g["presign"], atol=2e-4)
    for k in ("enc5", "enc8", "enc13"):          # after the linear-attention, space-attention and time-attention blocks
        assert torch.allclose(sample_like_golden(taps[k], g), g["taps"][k], atol=1e-4, rtol=1e-5), k


def test_restated_no_first_frame_matches_reference_golden():
    """video_contains_first_frame=False (M:1528-1537, M:1646-1647, M:1691): no front padding, no crop, frames % tdf == 0."""
    g = load_golden("mini_noff")
    assert g["first_frame"] is False
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    video = golden_video(g)
    taps = {}
    codes = orc.tokenize(video, taps=taps, video_contains_first_frame=False)
    assert torch.equal(codes, g["codes"]) and codes.shape[1] == video.shape[2] // 4
    dtaps = {}
    recon = orc.decode_from_code_indices(codes, taps=dtaps, video_contains_first_frame=False)
    assert recon.shape == video.shape
    assert torch.allclose(recon, g["recon"], atol=2e-5, rtol=1e-5)
    for k, ref in g["taps"].items():
        got = taps.get(k, dtaps.get(k))
        assert torch.allclose(sample_like_golden(got, g), ref, atol=2e-5, rtol=1e-5), k
    with pytest.raises(AssertionError):
        orc.tokenize(video)                      # 8 frames with a first frame: (8 - 1) % 4 != 0  (M:1691)


@pytest.mark.parametrize("mode", ["reflect", "replicate", "circular"])
def test_restated_pad_modes_match_reference_goldens(mode):
    """pad_mode of conv_in / conv_out (M:925-927, M:1109, M:1127)."""
    g = load_golden("pad_" + mode)
    assert g["kwargs"]["pad_mode"] == mode
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    codes = orc.tokenize(golden_video(g))
    assert torch.equal(codes, g["codes"])
    assert torch.allclose(orc.decode_from_code_indices(codes), g["recon"], atol=2e-5, rtol=1e-5)


def test_restated_cond_residual_matches_reference_golden():
    """SURVEY 8f N1 groundwork: the conditioned residual unit (ResidualUnitMod / Conv3DMod, M:680-753, M:946-988) and the
    conditioning stems (M:1344-1352), pinned to the reference before any kernel is written for it."""
    g = load_golden("mini_cond")
    orc = build_oracle_from_golden(g)
    video, cond = golden_video(g), g["cond"]
    taps = {}
    codes = orc.tokenize(video, taps=taps, cond=cond)
    assert torch.equal(codes, g["codes"])
    for k, ref in g["taps"].items():
        if k.startswith("enc") and k != "enc_cond_in":
            assert torch.allclose(sample_like_golden(taps[k], g), ref, atol=2e-5, rtol=1e-5), k
    assert torch.allclose(orc._cond_in(cond, "encoder"), g["taps"]["enc_cond_in"], atol=1e-6)
    dtaps = {}
    recon = orc.decode_from_code_indices(codes, taps=dtaps, cond=cond)
    assert torch.allclose(recon, g["recon"], atol=2e-5, rtol=1e-5)
    for k, ref in g["taps"].items():
        if k.startswith("dec"):
            assert torch.allclose(sample_like_golden(dtaps[k], g), ref, atol=2e-5, rtol=1e-5), k
    assert torch.equal(orc.forward(video, return_recon=True, cond=cond), recon)          # README.md:85-90 with cond
    # the modulation really depends on cond, per clip
    other = orc.tokenize(video, cond=cond.flip(0))
    assert not torch.equal(other, codes)
    with pytest.raises(AssertionError):
        orc.tokenize(video)                                                           # M:1542


def test_restated_separate_first_frame_encoding_matches_reference_golden():
    """SURVEY 8f N3 groundwork: separate_first_frame_encoding (first frame through its own 2-D convs, M:1553-1561,
    M:1633-1639), pinned to the reference."""
    g = load_golden("mini_sff")
    orc = build_oracle_from_golden(g)
    video = golden_video(g)
    taps, dtaps = {}, {}
    codes = orc.tokenize(video, taps=taps)
    assert torch.equal(codes, g["codes"])
    recon = orc.decode_from_code_indices(codes, taps=dtaps)
    assert torch.allclose(recon, g["recon"], atol=2e-5, rtol=1e-5)
    for k, ref in g["taps"].items():
        src = taps if (k.startswith("enc") or k == "conv_in") else dtaps
        if k == "conv_in":
            continue        # the reference's conv_in hook sees only frames 1.. (the first frame bypasses it)
        assert torch.allclose(sample_like_golden(src[k], g), ref, atol=2e-5, rtol=1e-5), k
    assert torch.equal(orc.forward(video, return_recon=True), recon)
    # after the input convs the first real frame depends on the first input frame only (2-D path)
    v2 = video.clone()
    v2[:, :, 1:] += 1.0
    t2 = {}
    orc.encode(v2, taps=t2)
    tp = orc.time_padding
    assert torch.equal(t2["conv_in"][:, :, :tp + 1], taps["conv_in"][:, :, :tp + 1])
    assert not torch.equal(t2["conv_in"][:, :, tp + 1:], taps["conv_in"][:, :, tp + 1:])
    assert torch.count_nonzero(taps["conv_in"][:, :, :tp]) == 0                      # re-padded with zero frames (M:1561)


def test_modulated_conv_factorises_into_shared_weight_conv():
    """The mapping the GPU path uses for Conv3DMod (M:736-751): per-clip weights w * (cond + 1) * inv_norm never need
    to be materialised --  y[b, o] = inv_norm[b, o] * conv(x[b] * (cond[b] + 1), w)[o]  with
    inv_norm[b, o] = rsqrt(max(sum_i (cond[b, i] + 1)^2 * S[o, i], eps)),  S[o, i] = sum_taps w[o, i, :]^2 --
    i.e. the shared-weight causal conv with a per-(clip, channel) input scale and a per-(clip, channel) output scale."""
    from oracle.restated import causal_conv3d, conv3d_mod
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 8, 4, 6, 6, generator=g)
    cond = torch.randn(3, 8, generator=g)
    w = torch.randn(16, 8, 3, 3, 3, generator=g)
    ref = conv3d_mod(x, cond, w)
    S = (w ** 2).sum(dim=(2, 3, 4))                                             # (O, I)
    inv_norm = (((cond + 1.) ** 2) @ S.t()).clamp(min=1e-8).rsqrt()             # (B, O)
    got = causal_conv3d(x * (cond + 1.)[:, :, None, None, None], w, None) * inv_norm[:, :, None, None, None]
    assert torch.allclose(got, ref, atol=1e-5, rtol=1e-5)


def test_cond_layers_must_be_trailing_like_in_the_reference():
    """has_cond is never reset (M:1153, M:1318): a plain layer after a cond layer gets cond= and raises in the reference."""
    from oracle.restated import OracleTokenizer
    with pytest.raises(TypeError):
        OracleTokenizer({}, image_size=32, init_dim=16, codebook_size=1024, dim_cond=8,
                        layers=("cond_residual", "residual"))
    with pytest.raises(TypeError):       # the product rejects the same specs at construction
        build_product(dict(image_size=32, init_dim=16, codebook_size=1024, dim_cond=8, layers=("cond_residual", "residual")))
    m = build_product(dict(image_size=32, init_dim=16, codebook_size=1024, dim_cond=8, layers=("residual", "cond_residual")))
    assert m.has_cond


def test_readme_roundtrip_property():
    """README.md:85-90: decode_from_code_indices(tokenize(v)) == forward(v, return_recon=True)."""
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    v = golden_video(g)
    assert torch.equal(orc.decode_from_code_indices(orc.tokenize(v)), orc.forward(v, return_recon=True))


def test_flat_ids_decode_equals_4d():
    """M:1587-1591."""
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    codes = g["codes"]
    a = orc.decode_from_code_indices(codes)
    b = orc.decode_from_code_indices(codes.reshape(codes.shape[0], -1))
    assert torch.equal(a, b)


def test_temporal_causality_and_batch_independence():
    """SURVEY.md 4 items 2 and 4 on the restated oracle."""
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(model, g["kwargs"])
    v = golden_video(g)
    c0 = orc.tokenize(v)
    v2 = v.clone()
    v2[:, :, 5:] += 1.0
    c1 = orc.tokenize(v2)
    assert torch.equal(c0[:, :2], c1[:, :2])          # latent frames 0-1 unaffected by frames >= 5
    assert torch.equal(orc.tokenize(v[:1]), c0[:1])    # batch independence


def test_dead_layernorm_never_applied():
    """SURVEY.md 3.1: the final LayerNorm is in state_dict but zip() drops it (M:1565)."""
    g = load_golden("cfg1")
    model = build_product(g["kwargs"], g["wseed"])
    n = len(g["kwargs"]["layers"])
    assert f"encoder_layers.{n}.1.weight" in model.state_dict()
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    sd[f"encoder_layers.{n}.1.weight"] += 100.0
    from oracle.restated import OracleTokenizer
    orc = OracleTokenizer(sd, **g["kwargs"])
    assert torch.equal(orc.tokenize(golden_video(g)), g["codes"])


def grad_digest_close(g, dg, rtol, what, atol=0.0):
    """g: a gradient tensor; dg: the golden's digest of the reference's gradient (oracle/make_train_golden.grad_digest).
    atol: absolute slack for gradients that are mathematically zero (the bias of a softmax logit: SE to_k.bias) and hold
    only round-off noise in the reference."""
    flat = g.detach().reshape(-1).double().cpu()
    assert tuple(g.shape) == tuple(dg["shape"]), what
    n_err = max(0.0, abs(float(flat.norm()) - dg["norm"]) - atol) / max(dg["norm"], 1e-30)
    samp = flat[::dg["stride"]]
    s_err = max(0.0, float((samp - dg["sample"].double()).abs().max()) - atol) / (float(dg["sample"].double().abs().max()) + 1e-30)
    assert n_err < rtol and s_err < rtol, (what, n_err, s_err, dg["norm"])
    return max(n_err, s_err)


@pytest.mark.parametrize("name", ["mini_train", "mini_mc_train", "mini_fsq_train", "mini_gateloop_train", "mini_cond_train", "mini_sff_train", "pad_reflect_train", "pad_circular_train"])
def test_restated_loss_forward_and_gradients_match_reference_golden(name):
    """SURVEY 8f N2: the differentiable restatement of forward(return_loss=True) reproduces the reference's loss values (eval and
    train mode) and, through autograd, the reference's gradient of every parameter (tests/golden/mini_train.pt, made by the
    unmodified reference: oracle/make_train_golden.py)."""
    g = load_golden(name)
    model = build_product(g["kwargs"], g["wseed"])
    video = golden_video(g)
    orc = build_oracle(model, g["kwargs"])
    cond = g.get("cond")
    with torch.no_grad():
        ev = orc.loss_forward(video, train=False, cond=cond)
    assert abs(ev["total_loss"].item() - g["eval"]["total_loss"].item()) < 1e-6
    assert abs(ev["recon_loss"].item() - g["eval"]["recon_loss_only"].item()) < 1e-6
    assert ev["aux"].item() == 0.0 and g["eval"]["aux"].item() == 0.0
    assert (ev["recon"].mean(dim=(3, 4)) - g["eval"]["recon_mean"]).abs().max().item() < 1e-5

    for v in orc.sd.values():
        if v.is_floating_point():
            v.requires_grad_(True)
    tr = orc.loss_forward(video, train=True, cond=cond)
    gt = g["train"]
    for k in ("total_loss", "recon_loss", "aux", "per_sample_entropy", "batch_entropy", "commitment"):
        if k in gt:                      # the three LFQ terms do not exist for FSQ
            assert abs(float(tr[k].detach()) - float(gt[k])) < 2e-6 * max(1.0, abs(float(gt[k]))), k
    tr["total_loss"].backward()
    worst = 0.0
    gnorm = sum(d["norm"] ** 2 for d in gt["grads"].values() if d is not None) ** 0.5
    for k, dg in gt["grads"].items():
        if dg is None:                    # parameters the reference's forward never touches (dead LayerNorm, ...)
            assert k not in orc.sd or orc.sd[k].grad is None or float(orc.sd[k].grad.abs().max()) == 0.0, k
            continue
        worst = max(worst, grad_digest_close(orc.sd[k].grad, dg, 2e-3, k, atol=1e-7 * gnorm))   # fp32 round-off through 28 layers and the inv_temperature = 100 softmax
    print(f"worst relative gradient deviation vs the reference: {worst:.2e}")
