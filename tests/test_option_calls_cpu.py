"""Host-side premises of tests/test_option_calls_gpu.py, without a GPU: its configs (OPTION_CONFIGS, every non-default
constructor option at the README widths), and for each

  * the kernel Engine.conv_kernel picks for the option-specific calls -- the Conv3DMod convs (with oscale / the residual),
    the gateloop's qkva conv, conv_in and conv_out under a pad mode (their padded inputs, pad (0, 0, 0)), sff's four
    parts, noff's kw-packed conv_in and channels-first conv_out -- and the exact list of calls meant for the CUDA-core conv;
  * the number of calls of each kind its stages imply (expected_option_calls, which the GPU test asserts);
  * the slab plans of the replays the pipeline defects are planted in, whose last tile has a disjoint predecessor on its CTA;
  * the replay grid: exact accumulation at every GEMM depth these configs reach, and an oscale grid of positive dyadic
    values at most 1, so the replayed oscale product only rounds once."""
import ctypes as C

import pytest
import torch

from bench import WORKLOADS
from tests.test_bench_calls_cpu import N_SM, _gemm_depths, assert_replay_grid_exact
from tests.test_bench_calls_gpu import REPLAY_GRID, last_cta
from tests.util import README_LAYERS

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200.engine import Engine, pack_conv, pack_conv_in_kwpack

BF = torch.bfloat16
WIDTHS = dict(image_size=128, init_dim=64, max_dim=512)
SHORT = ("residual", "compress_space", "compress_time", "residual")
GATELOOP = ("residual", "compress_space", "gateloop_time", "compress_space", "gateloop_time", "compress_time", "gateloop_time")
# the conv roles meant for the CUDA-core conv: conv_in on 3 input channels when it does not take the kw-packed ingest
SIMT_ROLES = ("conv_in", "conv_in_first_frame")
OSCALE_CONTROL = "clip 0's oscale (inv_norm) used for another clip"

OPTION_CONFIGS = {
    "fsq": dict(kw=WORKLOADS["fsq"]["kw"], clips=4, frames=17, controls=("FSQ indices with the mixed-radix digits reversed",)),
    "cond_deep": dict(kw=dict(WIDTHS, codebook_size=1024, dim_cond=12, layers=README_LAYERS + ("cond_residual",)),
                      clips=4, frames=17, controls=(OSCALE_CONTROL,)),
    "cond_wide": dict(kw=dict(WIDTHS, codebook_size=1024, dim_cond=12, layers=("residual", "cond_residual")),
                      clips=2, frames=17, many_tiles=("oscale",), controls=(OSCALE_CONTROL,)),
    "gateloop": dict(kw=dict(WIDTHS, codebook_size=1024, layers=GATELOOP), clips=2, frames=17, many_tiles=("qkva",),
                     controls=("the gateloop output taken from the state before the update",)),
    "sff": dict(kw=dict(WIDTHS, codebook_size=1024, separate_first_frame_encoding=True, layers=README_LAYERS), clips=2,
                frames=17, simt=["conv_in_first_frame", "conv_in"], controls=("sff's first frame read from frame tp + 1",)),
    "pad_reflect": dict(kw=dict(WIDTHS, codebook_size=1024, pad_mode="reflect", layers=SHORT), clips=2, frames=17,
                        simt=["conv_in"], controls=("reflect padding that includes the edge pixel",)),
    "pad_replicate": dict(kw=dict(WIDTHS, codebook_size=1024, pad_mode="replicate", layers=SHORT), clips=2, frames=17,
                          simt=["conv_in"]),
    "pad_circular": dict(kw=dict(WIDTHS, codebook_size=1024, pad_mode="circular", layers=SHORT), clips=2, frames=17,
                         simt=["conv_in"]),
    # mini_mc's codebook: 2 codebooks of 2^8 codes
    "mc_spherical": dict(kw=dict(WIDTHS, codebook_size=256, num_codebooks=2, lfq_spherical=True, layers=SHORT), clips=2,
                         frames=17),
    "noff": dict(kw=dict(WIDTHS, codebook_size=1024, layers=README_LAYERS), clips=2, frames=16, ff=False),
}


def option_kw(name):
    return OPTION_CONFIGS[name]["kw"]


def expected_option_calls(m, ff=True):
    """Calls per kind one tokenize + decode_from_code_indices makes: conv_in and conv_out (two convs each with sff); per
    ResidualUnit the fused kernel (C = 64 / 128) or two convs and squeeze_excite_residual; per Conv3DMod (cond_residual)
    to_cond's dense_small, one mod_prepare + scale_channels and two convs, plus the two cond stems; one conv per sampler;
    the attention stages' projections, fc1 / fc2 and two rmsnorms; per gateloop rmsnorm, qkva and the scan; one mv2_pad_cl
    for conv_in and one for conv_out under a pad mode; the quantiser and its decode."""
    n = dict(conv=2, ru=0, se=0, rmsnorm=0, quantize=1, codes=1, dense=0, mod=0, gateloop=0, pad=0)
    if m.separate_first_frame_encoding and ff:
        n["conv"] += 2
    if m.conv_in.pad_mode != "constant":
        n["pad"] += 2
    if m.has_cond:
        n["dense"] += 2
    for st in list(m.stages) * 2:
        if st.kind == "residual":
            fused = st.dim in (64, 128)
            n["ru"] += st.count if fused else 0
            n["conv"] += 0 if fused else 2 * st.count
            n["se"] += 0 if fused else st.count
        elif st.kind == "cond_residual":
            n.update(conv=n["conv"] + 2, dense=n["dense"] + 1, mod=n["mod"] + 1)
        elif st.kind in ("compress_space", "compress_time"):
            n["conv"] += 1
        elif st.kind in ("attend_space", "attend_time", "linear_attend_space"):
            n["conv"] += 5 if st.kind == "linear_attend_space" else 4
            n["rmsnorm"] += 2
        elif st.kind == "gateloop_time":
            n.update(conv=n["conv"] + 1, rmsnorm=n["rmsnorm"] + 1, gateloop=n["gateloop"] + 1)
        else:
            raise AssertionError(st.kind)
    return n


def tap_boxes(Ho, Wo):
    """(bw, bh, bt) output box of the tap-wise wgmma kernel (tc_conv.cu tc_tile_box): 128 positions."""
    p2 = lambda v: 1 << (v - 1).bit_length()
    bw = min(128, p2(Wo))
    bh = min(128 // bw, p2(Ho))
    return bw, bh, 128 // (bw * bh)


def _meta_model(name):
    with torch.device("meta"):
        return VideoTokenizer(**option_kw(name))


def option_calls(name):
    """(role, x_shape, pack, conv keywords, kernel) of the option-specific convs of config `name`, in call order."""
    m, cfg = _meta_model(name), OPTION_CONFIGS[name]
    B, S, ff = cfg["clips"], m.image_size, cfg.get("ff", True)
    T = cfg["frames"] + (m.time_padding if ff else 0)
    cin, cout = m.conv_in.conv, m.conv_out.conv
    kt, kh, kw = cin.weight.shape[2:]
    calls = []
    if m.separate_first_frame_encoding:
        ffw = m.conv_in_first_frame
        calls += [("conv_in_first_frame", (B, 1, S, S, 3), pack_conv(ffw.weight, ffw.bias, BF), {}, "simt"),
                  ("conv_in", (B, cfg["frames"] - 1, S, S, 3), pack_conv(cin.weight, cin.bias, BF), {}, "simt")]
    elif m.conv_in.pad_mode != "constant":
        calls.append(("conv_in", (B, T + kt - 1, S + 2 * (kh // 2), S + 2 * (kw // 2), 3), pack_conv(cin.weight, cin.bias, BF),
                      dict(pad=(0, 0, 0), out_spatial=(T, S, S)), "simt"))
    else:
        pin = pack_conv_in_kwpack(cin.weight, cin.bias)
        calls.append(("conv_in_kw", (B, T, S, S, pin.Ci_tc), pin, dict(pad=(kt - 1, kh // 2, 0)), "slab"))
    C_ = cin.weight.shape[0]

    def stage(mod, st, x, dec):
        nonlocal T, S, C_
        if st.kind == "cond_residual":
            calls.append(("mod_conv3", x, pack_conv(mod.conv.weights, None, BF), dict(oscale=True), "slab"))
            calls.append(("mod_conv1", x, pack_conv(mod.conv_out.weight, mod.conv_out.bias, BF), dict(res=True), "slab"))
        elif st.kind == "gateloop_time":
            w = mod.fn.fn.to_qkva[0].weight
            calls.append(("qkva", x, pack_conv(w[:, :, None, None, None], None, BF), {}, "slab"))
        elif st.kind == "compress_space":
            S, C_ = (2 * S, mod.net[0].weight.shape[0] // 4) if dec else (S // 2, mod.conv.weight.shape[0])
        elif st.kind == "compress_time":
            T, C_ = (2 * T, mod.net[0].weight.shape[0] // 2) if dec else ((T - 1) // 2 + 1, mod.conv.weight.shape[0])

    for i, st in enumerate(m.stages):
        stage(m.encoder_layers[i], st, (B, T, S, S, C_), False)
    for j, st in enumerate(reversed(m.stages)):
        stage(m.decoder_layers[j], st, (B, T, S, S, C_), True)
    tp = m.time_padding if ff else 0
    kt, kh, kw = cout.weight.shape[2:]
    pko = pack_conv(cout.weight, cout.bias, BF)
    if m.separate_first_frame_encoding:
        fo = m.conv_out_first_frame
        calls += [("conv_out_first_frame", (B, 1, S, S, C_), pack_conv(fo.weight, fo.bias, BF), {}, "slab"),
                  ("conv_out", (B, T - tp - 1, S, S, C_), pko, {}, "slab")]
    elif m.conv_out.pad_mode != "constant":
        calls.append(("conv_out", (B, T + kt - 1, S + 2 * (kh // 2), S + 2 * (kw // 2), C_), pko,
                      dict(pad=(0, 0, 0), out_spatial=(T, S, S)), "tap"))
    else:
        calls.append(("conv_out", (B, T, S, S, C_), pko, dict(pad=(kt - 1 - tp, kh // 2, kw // 2), out_spatial=(T - tp, S, S),
                                                             out_cf=True), "slab"))
    return calls


def _engine():
    eng = Engine(None)
    eng.dtype = BF
    return eng


def _ta(eng, x_shape, pk, kw):
    kw = dict(kw)
    res, os = kw.pop("res", False), kw.pop("oscale", False)
    ta = eng._tc_args(x_shape, pk, res=torch.empty(1) if res else None, oscale=torch.empty(1) if os else None, **kw)
    ta.x = ta.w = ta.y = 1
    return ta


# the option-specific calls each config makes, (role, x_shape, kernel) in call order
OPTION_TABLE = {
    "fsq": [("conv_in_kw", (4, 20, 128, 128, 32), "slab"), ("conv_out", (4, 20, 128, 128, 64), "slab")],
    "cond_deep": [("conv_in_kw", (4, 20, 128, 128, 32), "slab")] + [("mod_conv3", (4, 5, 16, 16, 512), "slab"),
                                                                  ("mod_conv1", (4, 5, 16, 16, 512), "slab")] * 2 + [
        ("conv_out", (4, 20, 128, 128, 64), "slab")],
    "cond_wide": [("conv_in_kw", (2, 17, 128, 128, 32), "slab")] + [("mod_conv3", (2, 17, 128, 128, 64), "slab"),
                                                                  ("mod_conv1", (2, 17, 128, 128, 64), "slab")] * 2 + [
        ("conv_out", (2, 17, 128, 128, 64), "slab")],
    "gateloop": [("conv_in_kw", (2, 18, 128, 128, 32), "slab"), ("qkva", (2, 18, 64, 64, 128), "slab"),
                 ("qkva", (2, 18, 32, 32, 256), "slab"), ("qkva", (2, 9, 32, 32, 512), "slab"),
                 ("qkva", (2, 9, 32, 32, 512), "slab"), ("qkva", (2, 18, 32, 32, 256), "slab"),
                 ("qkva", (2, 18, 64, 64, 128), "slab"), ("conv_out", (2, 18, 128, 128, 64), "slab")],
    "sff": [("conv_in_first_frame", (2, 1, 128, 128, 3), "simt"), ("conv_in", (2, 16, 128, 128, 3), "simt"),
            ("conv_out_first_frame", (2, 1, 128, 128, 64), "slab"), ("conv_out", (2, 16, 128, 128, 64), "slab")],
    "mc_spherical": [("conv_in_kw", (2, 18, 128, 128, 32), "slab"), ("conv_out", (2, 18, 128, 128, 64), "slab")],
    "noff": [("conv_in_kw", (2, 16, 128, 128, 32), "slab"), ("conv_out", (2, 16, 128, 128, 64), "slab")],
}
for _m in ("reflect", "replicate", "circular"):      # conv_in and conv_out on their padded inputs
    OPTION_TABLE[f"pad_{_m}"] = [("conv_in", (2, 24, 134, 134, 3), "simt"), ("conv_out", (2, 20, 130, 130, 64), "tap")]


@pytest.mark.parametrize("name", list(OPTION_CONFIGS))
def test_option_call_kernels(name):
    """Each option-specific call runs the kernel of the table; the CUDA-core calls are exactly the config's named ones."""
    eng = _engine()
    calls = option_calls(name)
    got = [(role, x, eng.conv_kernel(_ta(eng, x, pk, kw), pk)) for role, x, pk, kw, _ in calls]
    assert got == [(role, x, kind) for role, x, _, _, kind in calls]
    assert got == OPTION_TABLE[name], got
    assert [r for r, _, k in got if k == "simt"] == OPTION_CONFIGS[name].get("simt", [])
    assert set(OPTION_CONFIGS[name].get("simt", [])) <= set(SIMT_ROLES)
    if name.startswith("pad_"):     # the pad-0 conv_out: a 130^2 input plane for a 128^2 output, 128 boxes of 128 x 1 x 1
        (_, x, pk, kw, _), = [c for c in calls if c[0] == "conv_out"]
        assert tap_boxes(*kw["out_spatial"][1:]) == (128, 1, 1) and x[2:4] == (130, 130)


COUNTS = {
    "fsq": dict(conv=70, ru=6, se=16, rmsnorm=12, quantize=1, codes=1, dense=0, mod=0, gateloop=0, pad=0),
    "cond_deep": dict(conv=74, ru=6, se=16, rmsnorm=12, quantize=1, codes=1, dense=4, mod=2, gateloop=0, pad=0),
    "cond_wide": dict(conv=6, ru=2, se=0, rmsnorm=0, quantize=1, codes=1, dense=4, mod=2, gateloop=0, pad=0),
    "gateloop": dict(conv=14, ru=2, se=0, rmsnorm=6, quantize=1, codes=1, dense=0, mod=0, gateloop=6, pad=0),
    "sff": dict(conv=72, ru=6, se=16, rmsnorm=12, quantize=1, codes=1, dense=0, mod=0, gateloop=0, pad=0),
    "mc_spherical": dict(conv=10, ru=2, se=2, rmsnorm=0, quantize=1, codes=1, dense=0, mod=0, gateloop=0, pad=0),
    "noff": dict(conv=70, ru=6, se=16, rmsnorm=12, quantize=1, codes=1, dense=0, mod=0, gateloop=0, pad=0),
}
for _m in ("reflect", "replicate", "circular"):
    COUNTS[f"pad_{_m}"] = dict(COUNTS["mc_spherical"], pad=2)


@pytest.mark.parametrize("name", list(OPTION_CONFIGS))
def test_option_call_counts(name):
    m = _meta_model(name)
    assert expected_option_calls(m, OPTION_CONFIGS[name].get("ff", True)) == COUNTS[name]


# (config, role, index among that role's calls) -> (total tiles, grid) on 132 SMs of the replays the defects are planted in
DEFECT_PLANS = {("cond_deep", "mod_conv3", 0): (160, 132), ("cond_wide", "mod_conv3", 0): (None, 132),
                ("gateloop", "qkva", 0): (None, 132)}


def test_defect_target_plans():
    """The defect targets plan more tiles than CTAs, and the schedule's last tile has a disjoint predecessor."""
    eng, lib = _engine(), _engine().lib
    out = (C.c_int32 * 6)()
    for (name, role, idx), (want_total, want_grid) in DEFECT_PLANS.items():
        _, x, pk, kw, kind = [c for c in option_calls(name) if c[0] == role][idx]
        assert kind == "slab"
        ta = _ta(eng, x, pk, kw)
        assert lib.mv2_tc_slab_plan(C.byref(ta), N_SM, out) == 0, lib.mv2_last_error()
        mw, bn, total, grid = out[0], out[1], out[3], out[4]
        assert grid == want_grid and total > grid and (want_total is None or total == want_total), (name, total, grid)
        if name in ("cond_wide", "gateloop"):
            assert total > 2 * grid, (name, total, grid)        # more than two tiles per CTA
        tiles, k = [], 0
        while True:
            assert lib.mv2_tc_slab_tile(C.byref(ta), N_SM, last_cta(total, grid), k, out) == 0
            if out[0] < 0:
                break
            tiles.append(tuple(out))
            k += 1
        assert len(tiles) >= 2 and tiles[-1][0] == total - 1, (name, tiles)
        (_, b0, t0, h0, w0, n0), (_, b1, t1, h1, w1, n1) = tiles[-2:]
        assert not (b0 == b1 and t0 == t1 and abs(h0 - h1) < 16 and abs(w0 - w1) < 8 * mw and abs(n0 - n1) < bn), (name, tiles[-2:])


def test_replay_grid_with_oscale_is_exact_at_every_depth():
    ks = sorted({k for name in OPTION_CONFIGS for k in _gemm_depths(option_kw(name))[1]})
    assert max(ks) == 27 * 512
    assert_replay_grid_exact(ks)
    # oscale in {1..n} / 2^e: positive, at most 1 and dyadic, so the replayed accumulator times oscale keeps the
    # accumulator's exponent range and rounds once in fp32 (the exact bound's 3 u (S |os| + |b|) covers it and the bias add)
    n, e = REPLAY_GRID["os"]
    assert n == 2 ** e and all(float(torch.tensor(v * 2.0 ** -e, dtype=torch.float32)) == v * 2.0 ** -e for v in range(1, n + 1))
