"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle and the
committed reference goldens.  Run on the H100 box:  python -m pytest tests -m gpu"""
import os

import pytest
import torch

from tests.util import build_oracle, build_product, golden_video, load_golden, sample_like_golden

pytestmark = pytest.mark.gpu

FP32_RECON_TOL = 1e-5     # fp32 path vs the fp32 reference, max-abs (outputs are O(1)): the north-star's 1e-5
FP32_TAP_TOL = 1e-5       # per-layer activations of the small configs
FP32_README_TAP_TOL = 5e-5  # README config, 28 layers deep with O(10) activations near the bottleneck


def _require_cuda():
    assert torch.cuda.is_available(), "gpu-marked test without a GPU"


def _report(name, **kw):
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/parity_report.txt", "a") as f:
        f.write(name + ": " + ", ".join(f"{k}={v}" for k, v in kw.items()) + "\n")


@pytest.mark.parametrize("name", ["cfg1", "mini", "mini_fsq", "mini_mc", "mini_mc_fsq"])
def test_fp32_bit_exact_codes_and_recon_vs_golden(name):
    """fp32 storage + fp32 FMA: code indices bit-exact vs the reference golden, per-layer taps and recon
    within fp32 round-off."""
    _require_cuda()
    g = load_golden(name)
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    video = golden_video(g).cuda()
    eng = model.engine
    eng.taps = {}
    codes = model.tokenize(video)
    enc_taps, eng.taps = eng.taps, {}
    recon = model.decode_from_code_indices(codes)
    dec_taps, eng.taps = eng.taps, None
    worst = 0.0
    for k, ref in g["taps"].items():
        got = enc_taps.get(k, dec_taps.get(k))
        assert got is not None, k
        err = (sample_like_golden(got, g) - ref).abs().max().item()
        worst = max(worst, err)
        assert err < FP32_TAP_TOL, (k, err)
    assert codes.dtype == g["codes"].dtype
    n_diff = (codes.cpu() != g["codes"]).sum().item()
    rerr = (recon.cpu() - g["recon"]).abs().max().item()
    _report(f"fp32/{name}", code_mismatches=n_diff, recon_maxabs=f"{rerr:.3e}", worst_tap=f"{worst:.3e}")
    assert n_diff == 0, f"{n_diff} code indices differ from the reference"
    assert rerr < FP32_RECON_TOL, rerr


def test_fp32_readme_config_vs_golden():
    """BASELINE configs[1] (README config), one clip, fp32 path vs the reference golden."""
    _require_cuda()
    g = load_golden("readme")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    video = golden_video(g).cuda()
    eng = model.engine
    eng.taps = {}
    x = eng.encode_cl(video)
    _, codes, pre = eng.quantize_cl(x, want_quantized=False, want_aux=True)
    taps, eng.taps = eng.taps, None
    worst = 0.0
    for k, ref in g["taps"].items():
        if k in taps:
            err = (sample_like_golden(taps[k], g) - ref).abs().max().item()
            worst = max(worst, err)
            assert err < FP32_README_TAP_TOL, (k, err)
    pre_err = (pre.cpu().reshape(g["presign"].shape) - g["presign"]).abs().max().item()
    n_diff = (codes.cpu() != g["codes"]).sum().item()
    recon = model.decode_from_code_indices(g["codes"].cuda())
    rerr = (recon.cpu()[:, :, :, ::4, ::4] - g["recon_sample"]).abs().max().item()
    merr = (recon.cpu().mean(dim=(3, 4)) - g["recon_mean"]).abs().max().item()
    _report("fp32/readme", code_mismatches=n_diff, presign_maxabs=f"{pre_err:.3e}", recon_maxabs=f"{rerr:.3e}",
            recon_mean_err=f"{merr:.3e}", worst_enc_tap=f"{worst:.3e}")
    assert n_diff == 0
    assert rerr < FP32_RECON_TOL


@pytest.mark.parametrize("name", ["mini", "mini_fsq"])
def test_roundtrip_and_api_properties(name):
    """README.md:85-90 round trip, flat ids (M:1587-1591), image input (M:1681), batch independence."""
    _require_cuda()
    g = load_golden(name)
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    v = golden_video(g).cuda()
    codes = model.tokenize(v)
    a = model.decode_from_code_indices(codes)
    b = model(v, return_recon=True)
    assert torch.equal(a, b)
    c, r = model(v, return_codes=True, return_recon=True)
    assert torch.equal(c, codes) and torch.equal(r, a)
    flat = model.decode_from_code_indices(codes.reshape(codes.shape[0], -1))
    assert torch.equal(flat, a)
    assert torch.equal(model.tokenize(v[:1]), codes[:1])
    img_codes = model.tokenize(v[:, :, 0])
    assert img_codes.shape == (v.shape[0], 1, model.fmap_size, model.fmap_size)
    enc = model.encode(v)
    assert enc.shape[1] == model.quantizers.dim
    loss, rec = model(v, return_recon_loss_only=True)
    assert rec.shape == v.shape and loss.ndim == 0


# error budget of the bf16 product path + 50 %: (token mismatch rate, recon max-abs vs the fp32 reference)
# token flips on `mini` move between 2 and 6 of 96 tokens with the rounding points of a build; the reference's own bf16 run
# flips 5 of 96 (tests/golden/mini_bf16.pt): bound = 1.5x that
BF16_VS_FP32_BOUNDS = {"mini": (0.0834, 0.081), "mini_fsq": (0.125, 0.079)}


@pytest.mark.parametrize("name", ["mini", "mini_fsq"])
def test_bf16_path_vs_fp32_oracle(name):
    """bf16 storage / fp32 accumulate.  Protocol (SURVEY.md 8d): tokens whose code differs from the fp32
    oracle must have a small |pre-sign| margin there; decode is compared with identical codes."""
    _require_cuda()
    g = load_golden(name)
    cpu_model = build_product(g["kwargs"], g["wseed"])
    orc = build_oracle(cpu_model, g["kwargs"])
    v = golden_video(g)
    ref_codes = g["codes"]
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    codes = model.tokenize(v.cuda())
    mism = (codes.cpu() != ref_codes)
    rate = mism.float().mean().item()
    recon = model.decode_from_code_indices(ref_codes.cuda())
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    _report(f"bf16/{name}", token_mismatch_rate=f"{rate:.4f}", recon_maxabs=f"{rerr:.3e}")
    assert recon.dtype == torch.bfloat16
    rate_max, rerr_max = BF16_VS_FP32_BOUNDS[name]
    assert rate <= rate_max, rate
    assert rerr <= rerr_max, rerr
    if not g["kwargs"].get("use_fsq", False) and mism.any():
        margin = g["presign"].reshape(*ref_codes.shape, -1).abs().min(dim=-1).values
        assert margin[mism].max().item() < 0.07


@pytest.mark.parametrize("name", ["mini", "readme"])
def test_bf16_error_budget_vs_reference_bf16(name):
    """SURVEY 8d protocol (ii): the bf16 product path against the REFERENCE ITSELF run as ``model.bfloat16()``
    (tests/golden/<name>_bf16.pt, made by oracle/make_golden.py).  Both are compared with the fp32 reference golden,
    layer by layer; the product's error must stay within 1.5x of the reference's own bf16 error at every tap, its
    pre-sign deviation within 2x (max) / 1.5x (mean), its token mismatch rate and decode error (identical codes fed to both
    sides) within 1.5x."""
    _require_cuda()
    g32, g16 = load_golden(name), load_golden(name + "_bf16")
    assert g16["dtype"] == "bf16" and torch.equal(g16["codes_decoded"], g32["codes"])
    model = build_product(g32["kwargs"], g32["wseed"]).cuda().bfloat16()
    video = golden_video(g32).cuda()
    eng = model.engine
    eng.taps = {}
    x = eng.encode_cl(video)
    _, codes, pre = eng.quantize_cl(x, want_quantized=False, want_aux=True)
    taps, eng.taps = eng.taps, {}
    recon = model.decode_from_code_indices(g32["codes"].cuda())
    taps.update(eng.taps)
    eng.taps = None
    lines, worst_ratio = [], 0.0
    for k, ref32 in g32["taps"].items():
        got = sample_like_golden(taps[k], g32)
        e_prod, e_ref = (got - ref32).abs(), (g16["taps"][k] - ref32).abs()
        ratio = e_prod.mean().item() / (e_ref.mean().item() + 1e-9)
        worst_ratio = max(worst_ratio, ratio)
        lines.append(f"{k}:{e_prod.mean().item():.2e}/{e_ref.mean().item():.2e}")
        assert e_prod.mean().item() <= 1.5 * e_ref.mean().item() + 1e-5, (k, e_prod.mean().item(), e_ref.mean().item())
        assert e_prod.max().item() <= 2.0 * e_ref.max().item() + 1e-4, (k, e_prod.max().item(), e_ref.max().item())
    p32 = g32["presign"]
    dp_prod = (pre.cpu().reshape(p32.shape) - p32).abs()
    dp_ref = (g16["presign"] - p32).abs()
    mism_prod = (codes.cpu() != g32["codes"]).float().mean().item()
    mism_ref = (g16["codes"] != g32["codes"]).float().mean().item()
    flipped = (pre.cpu().reshape(p32.shape) > 0) != (p32 > 0)
    flip_margin = p32[flipped].abs().max().item() if flipped.any() else 0.0
    flipped_ref = (g16["presign"] > 0) != (p32 > 0)
    flip_margin_ref = p32[flipped_ref].abs().max().item() if flipped_ref.any() else 0.0
    if "recon" in g32:
        r_prod, r_ref = (recon.float().cpu() - g32["recon"]).abs(), (g16["recon"] - g32["recon"]).abs()
    else:
        r_prod = (recon.float().cpu()[:, :, :, ::4, ::4] - g32["recon_sample"]).abs()
        r_ref = (g16["recon_sample"] - g32["recon_sample"]).abs()
    _report(f"bf16-vs-ref-bf16/{name}", worst_tap_ratio=f"{worst_ratio:.2f}",
            presign_max=f"{dp_prod.max().item():.3e}/{dp_ref.max().item():.3e}",
            presign_mean=f"{dp_prod.mean().item():.3e}/{dp_ref.mean().item():.3e}",
            token_mismatch=f"{mism_prod:.4f}/{mism_ref:.4f}", flipped_bit_margin=f"{flip_margin:.3e}/{flip_margin_ref:.3e}",
            recon_max=f"{r_prod.max().item():.3e}/{r_ref.max().item():.3e}",
            recon_mean=f"{r_prod.mean().item():.3e}/{r_ref.mean().item():.3e}", taps="(product/reference-bf16 mean-abs vs fp32) " + " ".join(lines))
    assert dp_prod.max().item() <= 2.0 * dp_ref.max().item()
    assert dp_prod.mean().item() <= 1.5 * dp_ref.mean().item()
    assert mism_prod <= 1.5 * mism_ref + 1.0 / g32["codes"].numel()
    assert flip_margin <= 2.0 * max(flip_margin_ref, dp_ref.max().item())
    assert r_prod.max().item() <= 1.5 * r_ref.max().item()
    assert r_prod.mean().item() <= 1.5 * r_ref.mean().item()


def test_lfq_training_aux_terms_vs_oracle():
    """LFQ entropy / commitment terms (SURVEY Appendix A.1 steps 7-8) from the CUDA partial-sum kernel (+ the
    all-reduce path at world size 1) against the oracle, fp32."""
    _require_cuda()
    from oracle.restated import lfq_train_losses
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    codes, (ps, be, cm), aux = model.lfq_loss_breakdown(golden_video(g).cuda())
    assert torch.equal(codes.cpu(), g["codes"])
    rps, rbe, rcm, raux, _ = lfq_train_losses(g["presign"], 10)
    for got, ref in ((ps, rps), (be, rbe), (cm, rcm), (aux, raux)):
        assert abs(got.item() - ref.item()) <= 2e-4 * max(1.0, abs(ref.item())), (got.item(), ref.item())


def test_lfq_multi_codebook_spherical_aux_terms_vs_oracle():
    """num_codebooks = 2 + lfq_spherical (M:1057, M:1070): per-(token, codebook) entropies, per-codebook mean probabilities,
    commitment on the L2-normalised pre-sign values -- CUDA partial sums + finalize kernel against the oracle, fp32; plus the
    train-mode return_loss forward against the value the reference produced (tests/golden/mini_mc_train.pt)."""
    _require_cuda()
    from oracle.restated import lfq_train_losses
    g = load_golden("mini_mc")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    codes, (ps, be, cm), aux = model.lfq_loss_breakdown(golden_video(g).cuda())
    assert codes.shape[-1] == 2 and torch.equal(codes.cpu(), g["codes"])
    rps, rbe, rcm, raux, _ = lfq_train_losses(g["presign"], 8, nc=2)
    for got, ref in ((ps, rps), (be, rbe), (cm, rcm), (aux, raux)):
        assert abs(got.item() - ref.item()) <= 2e-4 * max(1.0, abs(ref.item())), (got.item(), ref.item())
    gt = load_golden("mini_mc_train")
    m2 = build_product(gt["kwargs"], gt["wseed"]).cuda().train()
    with torch.no_grad():
        total, bd = m2(golden_video(gt).cuda(), return_loss=True)
    assert abs(total.item() - gt["train"]["total_loss"].item()) < 1e-5
    assert abs(bd.lfq_aux_loss.item() - gt["train"]["aux"].item()) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cuda_graph_replay_equals_eager(dtype):
    """Opt-in CUDA-graph replay of the static launch plan returns exactly what the eager launches return."""
    _require_cuda()
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    vids = [golden_video(g).cuda() + 0.1 * i for i in range(4)]
    eager = [(model.tokenize(v), model(v, return_recon=True)) for v in vids]
    dec_eager = [model.decode_from_code_indices(c) for c, _ in eager]
    model.cuda_graphs = True
    model.pdl = True                        # programmatic dependent launch on top of graph replay
    for rep in range(2):
        for i, v in enumerate(vids):                # call 0 warms up, call 1 captures, later calls replay
            c = model.tokenize(v)
            r = model(v, return_recon=True)
            d = model.decode_from_code_indices(c)
            assert torch.equal(c, eager[i][0])
            assert torch.equal(r, eager[i][1])
            assert torch.equal(d, dec_eager[i])
    assert any(isinstance(e, tuple) for e in model._graphs.values()), "no graph was captured"


def test_bf16_readme_config_vs_reference_golden():
    """BASELINE configs[1] (README config) on the bf16 wgmma path against the fp32 reference golden.
    Protocol of SURVEY.md 8d: (i) tokens whose code differs from the fp32 reference must sit on a small |pre-sign|
    margin there (the reference's own bf16-vs-fp32 disagreement is 2-4 % of tokens, BASELINE.md 2);
    (ii) decode is compared with IDENTICAL codes fed to both sides."""
    _require_cuda()
    g = load_golden("readme")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    video = golden_video(g).cuda()
    codes = model.tokenize(video)
    eng = model.engine
    assert eng.simt_conv_calls == 0, "a convolution fell back to the CUDA-core path"
    mism = codes.cpu() != g["codes"]
    rate = mism.float().mean().item()
    margin = g["presign"].reshape(*g["codes"].shape, -1).abs().min(dim=-1).values
    worst_margin = margin[mism].max().item() if mism.any() else 0.0
    recon = model.decode_from_code_indices(g["codes"].cuda())
    rerr = (recon.float().cpu()[:, :, :, ::4, ::4] - g["recon_sample"]).abs()
    _report("bf16/readme", token_mismatch_rate=f"{rate:.4f}", worst_flipped_margin=f"{worst_margin:.3e}",
            recon_maxabs=f"{rerr.max().item():.3e}", recon_meanabs=f"{rerr.mean().item():.3e}")
    # error budget of the bf16 product path; the reference's own bf16 run: 5.2 % of tokens, margin 6.1e-2, recon 4.6e-2 / 8.1e-3
    assert rate < 0.04, rate
    assert worst_margin < 0.094, worst_margin
    assert rerr.max().item() < 0.057 and rerr.mean().item() < 0.0102


def test_bf16_tensor_core_path_vs_bf16_cuda_core_path():
    """Same bf16 storage / fp32 accumulate arithmetic on both paths: the wgmma kernels must agree with the CUDA-core
    kernels far more tightly than bf16 agrees with fp32."""
    _require_cuda()
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    v = golden_video(g).cuda()
    eng = model.engine
    eng.taps = {}
    c_tc = model.tokenize(v)
    taps_tc, eng.taps = eng.taps, {}
    eng.use_tc = False
    c_cc = model.tokenize(v)
    taps_cc, eng.taps = eng.taps, None
    eng.use_tc = True
    worst = {}
    for k in taps_tc:
        a, b = taps_tc[k], taps_cc[k]
        worst[k] = (a - b).abs().mean().item() / (b.abs().mean().item() + 1e-6)
    _report("bf16/tc_vs_cuda_core", **{k: f"{v:.4f}" for k, v in worst.items()},
            code_mismatch=f"{(c_tc != c_cc).float().mean().item():.4f}")
    # bf16 keeps 8 mantissa bits: two correct implementations with different fusion / accumulation order drift apart by
    # ~0.4 % per rounding point; the stack is ~30 layers deep
    for k, v in worst.items():
        assert v < 0.03, (k, v)
    # mini has 96 tokens x 10 sign bits with many pre-sign values within bf16 noise of zero: bound the flip rate loosely
    # and require that every flipped token sits on a small fp32 margin (a real defect flips confident tokens too)
    mism = (c_tc != c_cc).cpu()
    margin = g["presign"].reshape(*g["codes"].shape, -1).abs().min(dim=-1).values
    assert mism.float().mean().item() < 0.15
    assert (margin[mism].max().item() if mism.any() else 0.0) < 0.1


WIDE_KW = dict(image_size=32, init_dim=128, max_dim=1024, codebook_size=4096,
               layers=("residual", "compress_space", ("consecutive_residual", 2), "linear_attend_space", "compress_space",
                       "residual", "attend_space", "compress_time", "residual", "compress_space", "residual", "attend_time"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_wide_channel_config_vs_oracle(dtype):
    """Channel widths of BASELINE configs[3] (max_dim 1024: 128 -> 256 -> 512 -> 1024) at toy spatial size, checked live
    against the CPU oracle: exercises the 4-n-tile slab path, the 32-wide SE / norm vector variants and a 12-bit LFQ."""
    _require_cuda()
    cpu_model = build_product(WIDE_KW, 3)
    orc = build_oracle(cpu_model, WIDE_KW)
    from oracle import weights as W
    v = W.synth_video(2, 3, 5, 32, seed=77)
    ref_codes, pre = orc.tokenize(v, return_presign=True)
    ref_recon = orc.decode_from_code_indices(ref_codes)
    model = build_product(WIDE_KW, 3).cuda().to(dtype)
    codes = model.tokenize(v.cuda())
    recon = model.decode_from_code_indices(ref_codes.cuda())
    mism = codes.cpu() != ref_codes
    rerr = (recon.float().cpu() - ref_recon).abs()
    _report(f"wide/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism.float().mean().item():.4f}",
            recon_maxabs=f"{rerr.max().item():.3e}", min_margin=f"{pre.abs().min().item():.2e}")
    if dtype == torch.float32:
        margin = pre.reshape(*ref_codes.shape, -1).abs().min(dim=-1).values
        assert (not mism.any()) or margin[mism].max().item() < 2e-5      # only sign tests on a ~1e-5 margin may flip
        assert rerr.max().item() < 2e-5
    else:
        assert mism.float().mean().item() <= 0.0834      # at most 8 of 96 tokens
        assert rerr.mean().item() < 0.012 and rerr.max().item() < 0.06


@pytest.mark.parametrize("lanes", [1, 2, 3])
@pytest.mark.parametrize("graphs", [False, True])
def test_host_round_trip_matches_direct_calls(graphs, lanes):
    """HostRoundTrip (pinned host buffers, copies overlapped on side streams) returns exactly what tokenize /
    decode_from_code_indices return for device inputs, for every in-flight slot and across slot reuse."""
    _require_cuda()
    from magvit2_pytorch_b200 import HostRoundTrip
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    vids = [(golden_video(g) + 0.05 * i).pin_memory() for i in range(5)]
    want = []
    for v in vids:
        c = model.tokenize(v.cuda())
        want.append((c.cpu(), model.decode_from_code_indices(c).cpu()))
    model.cuda_graphs = graphs
    hrt = HostRoundTrip(model, depth=max(2, lanes), lanes=lanes)
    outs = [(torch.empty_like(want[0][0]).pin_memory(), torch.empty_like(want[0][1]).pin_memory()) for _ in vids]
    for rep in range(2):
        evs = [hrt.submit(v, oc, ov) for v, (oc, ov) in zip(vids, outs)]
        hrt.wait(evs[-1])
        hrt.synchronize()
        for (oc, ov), (wc, wv) in zip(outs, want):
            assert torch.equal(oc, wc)
            assert torch.equal(ov, wv)
    with pytest.raises(ValueError):
        hrt.submit(vids[0].clone(), outs[0][0], outs[0][1])      # not pinned


@pytest.mark.parametrize("graphs", [False, True])
def test_stream_lanes_match_serial_calls(graphs):
    """StreamLanes: calls issued round-robin on several CUDA streams (each lane replaying its own graph instances) return
    exactly what the same calls return one after the other on the current stream."""
    _require_cuda()
    from magvit2_pytorch_b200 import StreamLanes
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    vids = [(golden_video(g) + 0.03 * i).cuda() for i in range(7)]

    def step(v):
        c = model.tokenize(v)
        return c, model.decode_from_code_indices(c)

    want = [step(v) for v in vids]
    model.cuda_graphs = graphs
    lanes = StreamLanes(model, 3)
    for rep in range(3):                       # plain call, capture, replay on every lane
        got = [lanes.run(step, v)[0] for v in vids]
        lanes.join()
        torch.cuda.synchronize()
        for (gc, gv), (wc, wv) in zip(got, want):
            assert torch.equal(gc, wc)
            assert torch.equal(gv, wv)
    if graphs:
        assert len({k[3] for k in model._graphs}) == 3       # one set of graph instances per lane
    assert model._lane == 0


def test_copy_for_eval_after_graph_capture_and_repack():
    """Captured CUDA graphs (static buffers, private pools) belong to one instance and one parameter version:
    copy_for_eval() / deepcopy / pickling start without them, and a re-pack drops the stale entries."""
    _require_cuda()
    import copy
    import pickle
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    v = golden_video(g).cuda()
    want = model.tokenize(v)
    model.cuda_graphs = True
    for _ in range(3):
        assert torch.equal(model.tokenize(v), want)
    assert any(isinstance(e, tuple) for e in model._graphs.values())
    c = model.copy_for_eval()
    assert c._graphs == {} and c._engine is None
    assert torch.equal(c.tokenize(v), want)
    d = copy.deepcopy(model)
    assert d._graphs == {}
    p = pickle.loads(pickle.dumps(model))
    assert p._graphs == {} and torch.equal(p.tokenize(v), want)
    # the cpu() / to(dev) round trip inside copy_for_eval re-packed the original: its old graphs must be gone after one call
    sig_before = {k[1] for k in model._graphs}
    assert torch.equal(model.tokenize(v), want)
    assert all(k[1] == model.engine._sig_id for k in model._graphs), (sig_before, model.engine._sig_id)


def test_device_mismatch_raises_cleanly():
    """CPU (or other-device) inputs raise a RuntimeError instead of handing a foreign pointer to the kernels."""
    _require_cuda()
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    with pytest.raises(RuntimeError):
        model.decode_from_code_indices(g["codes"])                  # CPU codes
    with pytest.raises(RuntimeError):
        model.decode(torch.zeros(1, model.quantizers.dim, 3, 4, 4))  # CPU latents
    with pytest.raises(AssertionError):
        model.decode(torch.zeros(1, 7, 3, 4, 4, device="cuda"))      # wrong channel count
    with pytest.raises(RuntimeError):
        model.tokenize(golden_video(g))                             # CPU video


def test_model_on_non_current_device():
    """The C ABI launches on the current device: the host class must make its own device current (2+ GPUs only)."""
    _require_cuda()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = load_golden("mini")
    v = golden_video(g)
    for dt in (torch.float32, torch.bfloat16):
        m0 = build_product(g["kwargs"], g["wseed"]).to("cuda:0").to(dt)
        m1 = build_product(g["kwargs"], g["wseed"]).to("cuda:1").to(dt)
        torch.cuda.set_device(0)
        c0 = m0.tokenize(v.to("cuda:0"))
        c1 = m1.tokenize(v.to("cuda:1"))           # current device is 0
        assert c1.device == torch.device("cuda:1")
        assert torch.equal(c0.cpu(), c1.cpu())
        r1 = m1.decode_from_code_indices(c1)
        assert torch.equal(m0.decode_from_code_indices(c0).cpu(), r1.cpu())


@pytest.mark.parametrize("name", ["cfg4", "fsq"])
def test_full_size_configs_vs_reference_goldens(name):
    """BASELINE configs[3] (image 256, max_dim 1024, attention-heavy) and configs[4] (FSQ) at FULL size against the
    reference goldens: fp32 path bit-exact codes + recon within 1e-5-class tolerance; bf16 path inside the reference's own
    bf16 error budget (1.5x, per tap and end to end), decode with identical codes."""
    _require_cuda()
    g32, g16 = load_golden(name), load_golden(name + "_bf16")
    rs = g32.get("recon_stride", 4)
    video = golden_video(g32).cuda()
    # ---- fp32 path ----
    model = build_product(g32["kwargs"], g32["wseed"]).cuda()
    codes = model.tokenize(video)
    n_diff = (codes.cpu() != g32["codes"]).sum().item()
    recon = model.decode_from_code_indices(g32["codes"].cuda())
    rerr = (recon.cpu()[:, :, :, ::rs, ::rs] - g32["recon_sample"]).abs().max().item()
    _report(f"fp32/{name}", code_mismatches=n_diff, recon_maxabs=f"{rerr:.3e}")
    assert codes.dtype == g32["codes"].dtype
    if name == "fsq":
        # FSQ rounds |bounded| values at half-integers: a 1e-6 fp32 difference can move a value across .5
        assert n_diff <= 2, n_diff
    else:
        assert n_diff == 0, n_diff
    assert rerr < 2e-5, rerr
    del model
    # ---- bf16 path vs the reference's own bf16 run ----
    model = build_product(g32["kwargs"], g32["wseed"]).cuda().bfloat16()
    eng = model.engine
    eng.taps = {}
    x = eng.encode_cl(video)
    _, codes16, _ = eng.quantize_cl(x, want_quantized=False)
    taps, eng.taps = eng.taps, {}
    recon16 = model.decode_from_code_indices(g32["codes"].cuda())
    taps.update(eng.taps)
    eng.taps = None
    assert eng.simt_conv_calls == 0, "a convolution fell back to the CUDA-core path"
    worst = 0.0
    for k, ref32 in g32["taps"].items():
        e_prod = (sample_like_golden(taps[k], g32) - ref32).abs().mean().item()
        e_ref = (g16["taps"][k] - ref32).abs().mean().item()
        worst = max(worst, e_prod / (e_ref + 1e-9))
        assert e_prod <= 1.5 * e_ref + 1e-5, (k, e_prod, e_ref)
    mism_prod = (codes16.cpu() != g32["codes"]).float().mean().item()
    mism_ref = (g16["codes"] != g32["codes"]).float().mean().item()
    r_prod = (recon16.float().cpu()[:, :, :, ::rs, ::rs] - g32["recon_sample"]).abs()
    r_ref = (g16["recon_sample"] - g32["recon_sample"]).abs()
    _report(f"bf16-vs-ref-bf16/{name}", worst_tap_ratio=f"{worst:.2f}", token_mismatch=f"{mism_prod:.4f}/{mism_ref:.4f}",
            recon_max=f"{r_prod.max().item():.3e}/{r_ref.max().item():.3e}", recon_mean=f"{r_prod.mean().item():.3e}/{r_ref.mean().item():.3e}")
    assert mism_prod <= 1.5 * mism_ref + 2.0 / g32["codes"].numel()
    assert r_prod.max().item() <= 1.5 * r_ref.max().item() and r_prod.mean().item() <= 1.5 * r_ref.mean().item()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_video_without_first_frame_vs_reference_golden(dtype):
    """video_contains_first_frame=False (M:1528-1537, M:1646-1647, M:1691) through encode / forward / decode_from_code_indices."""
    _require_cuda()
    g = load_golden("mini_noff")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    v = golden_video(g).cuda()
    codes = model(v, return_codes=True, video_contains_first_frame=False)
    recon = model.decode_from_code_indices(g["codes"].cuda(), video_contains_first_frame=False)
    assert recon.shape == v.shape and codes.shape == g["codes"].shape
    c2, r2 = model(v, return_codes=True, return_recon=True, video_contains_first_frame=False)
    assert torch.equal(c2, codes)
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    mism = (codes.cpu() != g["codes"]).float().mean().item()
    _report(f"noff/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism:.4f}", recon_maxabs=f"{rerr:.3e}")
    if dtype == torch.float32:
        assert mism == 0 and rerr < FP32_RECON_TOL
        assert torch.equal(r2, recon)
    else:
        assert mism <= 0.0834 and rerr < 0.081
    with pytest.raises(AssertionError):
        model.tokenize(v)                        # 8 frames WITH a first frame: (8 - 1) % 4 != 0
    model.cuda_graphs = True
    for _ in range(3):
        assert torch.equal(model(v, return_codes=True, video_contains_first_frame=False), codes)


@pytest.mark.parametrize("graphs", [False, True])
def test_train_mode_forward_world1(graphs):
    """``model.train()`` forward (reference M:1705 in training mode): codes identical to eval, reconstruction from q, and the
    LFQ auxiliary terms (world size 1 here; tests/test_dist_gpu.py runs the all-reduce over 2 GPUs) vs the oracle."""
    _require_cuda()
    from oracle.restated import lfq_train_losses
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    v = golden_video(g).cuda()
    want_recon = model.decode_from_code_indices(g["codes"].cuda())
    model.train()
    model.cuda_graphs = graphs
    for _ in range(3 if graphs else 1):
        codes, recon = model(v, return_codes=True, return_recon=True)
        ps, be, cm = model.quantizer_loss_breakdown
    assert torch.equal(codes.cpu(), g["codes"])
    assert torch.equal(recon, want_recon)
    rps, rbe, rcm, raux, _ = lfq_train_losses(g["presign"], 10)
    for got, ref in ((ps, rps), (be, rbe), (cm, rcm), (model.quantizer_aux_loss, raux)):
        assert abs(got.item() - ref.item()) <= 2e-4 * max(1.0, abs(ref.item())), (got.item(), ref.item())
    only_codes = model(v, return_codes=True)
    assert torch.equal(only_codes, codes)
    assert torch.equal(model.tokenize(v), codes) and not model.training          # tokenize() switches to eval (M:1653)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cond_residual_vs_reference_golden(dtype):
    """SURVEY 8f N1: cond_residual (ResidualUnitMod / Conv3DMod, M:680-753, M:946-988) on the device -- input-channel
    modulation + shared-weight conv + per-(clip, channel) demodulation in the epilogue -- against the reference golden."""
    _require_cuda()
    g = load_golden("mini_cond")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    v, cond = golden_video(g).cuda(), g["cond"].cuda()
    eng = model.engine
    eng.taps = {}
    codes = model(v, cond=cond, return_codes=True)
    enc_taps, eng.taps = eng.taps, {}
    recon = model.decode_from_code_indices(g["codes"].cuda(), cond=cond)
    dec_taps, eng.taps = eng.taps, None
    mism = (codes.cpu() != g["codes"]).float().mean().item()
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    worst = 0.0
    for k, ref in g["taps"].items():
        got = enc_taps.get(k, dec_taps.get(k))
        if got is None:
            continue
        worst = max(worst, (sample_like_golden(got, g) - ref).abs().max().item())
    _report(f"cond/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism:.4f}", recon_maxabs=f"{rerr:.3e}", worst_tap=f"{worst:.3e}")
    if dtype == torch.float32:
        assert mism == 0 and rerr < FP32_RECON_TOL and worst < FP32_TAP_TOL
        c2, r2 = model(v, cond=cond, return_codes=True, return_recon=True)
        assert torch.equal(c2, codes) and torch.equal(r2, recon)
        other = model(v, cond=cond.flip(0), return_codes=True)
        assert not torch.equal(other, codes)                       # the modulation really depends on cond, per clip
    else:
        assert mism <= 0.1 and rerr < 0.1
    with pytest.raises(AssertionError):
        model(v, return_codes=True)                                # cond missing (M:1542)
    model.cuda_graphs = True
    for _ in range(3):
        assert torch.equal(model(v, cond=cond, return_codes=True), codes)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_separate_first_frame_encoding_vs_reference_golden(dtype):
    """SURVEY 8f N3: separate_first_frame_encoding (M:1113-1120, M:1553-1561, M:1633-1639) against the reference golden."""
    _require_cuda()
    g = load_golden("mini_sff")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    v = golden_video(g).cuda()
    eng = model.engine
    eng.taps = {}
    codes = model.tokenize(v)
    enc_taps, eng.taps = eng.taps, {}
    recon = model.decode_from_code_indices(g["codes"].cuda())
    dec_taps, eng.taps = eng.taps, None
    mism = (codes.cpu() != g["codes"]).float().mean().item()
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    worst = 0.0
    for k, ref in g["taps"].items():
        got = enc_taps.get(k, dec_taps.get(k))
        if got is not None and sample_like_golden(got, g).shape == ref.shape:     # (the reference's conv_in hook only sees frames 1..)
            worst = max(worst, (sample_like_golden(got, g) - ref).abs().max().item())
    _report(f"sff/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism:.4f}", recon_maxabs=f"{rerr:.3e}", worst_tap=f"{worst:.3e}")
    assert recon.shape == v.shape
    if dtype == torch.float32:
        assert mism == 0 and rerr < FP32_RECON_TOL and worst < FP32_TAP_TOL
        assert torch.equal(model(v, return_recon=True), model.decode_from_code_indices(codes))
        img = model.tokenize(v[:, :, 0])                  # single image: only the first-frame convs run
        assert img.shape == (v.shape[0], 1, model.fmap_size, model.fmap_size)
    else:
        assert mism <= 0.1 and rerr < 0.1


@pytest.mark.parametrize("mode", ["reflect", "replicate", "circular"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_pad_modes_vs_reference_goldens(mode, dtype):
    """pad_mode != 'constant' on conv_in / conv_out (M:925-927: F.pad(..., mode) before the conv) vs the reference goldens."""
    _require_cuda()
    g = load_golden("pad_" + mode)
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    v = golden_video(g).cuda()
    codes = model.tokenize(v)
    recon = model.decode_from_code_indices(g["codes"].cuda())
    mism = (codes.cpu() != g["codes"]).float().mean().item()
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    _report(f"pad_{mode}/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism:.4f}", recon_maxabs=f"{rerr:.3e}")
    if dtype == torch.float32:
        assert mism == 0 and rerr < FP32_RECON_TOL
    else:
        assert mism <= 0.08 and rerr < 0.08


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_readme_config_batch_independence(dtype):
    """Eval forward has no cross-sample op (SURVEY 8e): a 3-clip batch must give exactly the per-clip results, also for the
    persistent-kernel tile schedules, the fused ResidualUnit records and the SE chunking, which all depend on the batch size."""
    _require_cuda()
    g = load_golden("readme")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    from oracle import weights as W
    v = W.synth_video(3, 3, 17, 128, seed=4321).cuda()
    codes = model.tokenize(v)
    recon = model.decode_from_code_indices(codes)
    for i in range(3):
        ci = model.tokenize(v[i:i + 1])
        assert torch.equal(ci, codes[i:i + 1]), i
        assert torch.equal(model.decode_from_code_indices(ci), recon[i:i + 1]), i


@pytest.mark.gpu
def test_return_loss_forward_vs_reference_golden():
    """forward(video, return_loss=True) / return_recon_loss_only (reference M:1722-1727, M:1868-1896; use_gan=False,
    perceptual_loss_weight=0) against the values the unmodified reference produced (tests/golden/mini_train.pt), eval and
    train mode, fp32; bf16 against the same values at the bf16 error budget."""
    _require_cuda()
    from magvit2_pytorch_b200.video_tokenizer import LossBreakdown
    g = load_golden("mini_train")
    video = golden_video(g).cuda()
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    total, bd = model(video, return_loss=True)
    assert isinstance(bd, LossBreakdown) and bd.quantizer_loss_breakdown is None and bd.multiscale_gen_losses == []
    assert abs(total.item() - g["eval"]["total_loss"].item()) < 2e-6
    assert abs(bd.recon_loss.item() - g["eval"]["recon_loss"].item()) < 2e-6 and float(bd.lfq_aux_loss) == 0.0
    rl, recon = model(video, return_recon_loss_only=True)
    assert abs(rl.item() - g["eval"]["recon_loss_only"].item()) < 2e-6
    assert (recon.mean(dim=(3, 4)).cpu() - g["eval"]["recon_mean"]).abs().max().item() < 1e-5
    assert abs(rl.item() - torch.nn.functional.mse_loss(video, recon).item()) < 1e-6

    model.train()
    with torch.no_grad():
        total, bd = model(video, return_loss=True)
    gt = g["train"]
    assert abs(total.item() - gt["total_loss"].item()) < 1e-5
    assert abs(bd.recon_loss.item() - gt["recon_loss"].item()) < 1e-5
    assert abs(bd.lfq_aux_loss.item() - gt["aux"].item()) < 1e-5
    ps, be, cm = bd.quantizer_loss_breakdown
    assert abs(ps.item() - gt["per_sample_entropy"].item()) < 1e-5
    assert abs(be.item() - gt["batch_entropy"].item()) < 1e-5
    assert abs(cm.item() - gt["commitment"].item()) < 1e-5

    m16 = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16().eval()
    t16, bd16 = m16(video.bfloat16(), return_loss=True)
    assert t16.dtype == torch.bfloat16
    assert abs(t16.float().item() - g["eval"]["total_loss"].item()) < 0.05 * g["eval"]["total_loss"].item()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_uint8_frames_are_normalised_like_the_data_loaders(dtype):
    """uint8 frames (what a video decoder delivers) are accepted by the layout-in kernels and normalised x / 255 there, exactly as
    the reference's loaders do on the host (data.py:103 ToTensor, data.py:188): tokens and reconstruction are bit-identical to
    feeding ``frames.float() / 255``."""
    _require_cuda()
    g = load_golden("mini")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    gen = torch.Generator().manual_seed(3)
    frames = torch.randint(0, 256, tuple(g["video_shape"]), generator=gen, dtype=torch.uint8).cuda()
    as_float = frames.float() / 255.
    c8, r8 = model(frames, return_codes=True, return_recon=True)
    cf, rf = model(as_float, return_codes=True, return_recon=True)
    assert torch.equal(c8, cf) and torch.equal(r8, rf)
    l8, _ = model(frames, return_recon_loss_only=True)
    lf, _ = model(as_float, return_recon_loss_only=True)
    assert l8.item() == lf.item()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gateloop_time_vs_reference_golden(dtype):
    """SURVEY 8f N3: gateloop_time (ToTimeSequence(Residual(SimpleGateLoopLayer)), M:178-191, M:1216-1222) on the device -- RMSNorm,
    the 1x1x1 projection kernels and mv2_gateloop_scan -- against the golden the reference produced (through the restated
    SimpleGateLoopLayer of oracle/shims/gateloop.py: the dependency's arithmetic is "parity unpinned")."""
    _require_cuda()
    g = load_golden("mini_gateloop")
    model = build_product(g["kwargs"], g["wseed"]).cuda().to(dtype)
    v = golden_video(g).cuda()
    eng = model.engine
    eng.taps = {}
    codes = model.tokenize(v)
    enc_taps, eng.taps = eng.taps, {}
    recon = model.decode_from_code_indices(g["codes"].cuda())
    dec_taps, eng.taps = eng.taps, None
    mism = (codes.cpu() != g["codes"]).float().mean().item()
    rerr = (recon.float().cpu() - g["recon"]).abs().max().item()
    worst = 0.0
    for k, ref in g["taps"].items():
        got = enc_taps.get(k, dec_taps.get(k))
        if got is None:
            continue
        worst = max(worst, (sample_like_golden(got, g) - ref).abs().max().item())
    _report(f"gateloop/{str(dtype).split('.')[-1]}", token_mismatch_rate=f"{mism:.4f}", recon_maxabs=f"{rerr:.3e}", worst_tap=f"{worst:.3e}")
    if dtype == torch.float32:
        assert mism == 0 and rerr < FP32_RECON_TOL and worst < FP32_TAP_TOL
    else:
        assert mism <= 0.1 and rerr < 0.1
    model.cuda_graphs = True
    for _ in range(3):
        assert torch.equal(model.tokenize(v), codes)
