"""Host-side premises of tests/test_train_calls_gpu.py, without a GPU, for the README training step's discriminator and VGG
(VideoTokenizer(image_size=128, init_dim=64, max_dim=512, ..., vgg=build_vgg(VGG16_CFG, 4096)), 4 clips, one frame per
clip through each network):

  * the kernel Engine.conv_kernel picks for every engine conv the discriminator (gan.DiscrRunner) and the VGG
    (vgg.VggRunner) run, forward and data gradient, derived from the modules.  The discriminator's widths are 3 -> 512 ->
    512 ... 512 (its `dim` is the tokenizer's last stage width, 512), six blocks down to a 4 x 4 map;
  * the number of calls of each kind one forward / backward makes, from the module structure;
  * the exact-replay grid at every GEMM depth these calls reach (up to 8192 = 512 channels x 16 taps): every product
    and partial sum is a multiple of 2^-8 below 2^14, so an fp32 accumulation is exact in any order.  Checked by the
    arithmetic and by fp32 sums in shuffled orders against float64.

readme_table() is the table the GPU test asserts its recorded calls against: a later dispatch change cannot silently move one of
these calls off the kernel the GPU test checks.

tokenizer_table() / tokenizer_counts() are the same for the tokenizer's own calls in that step
(tests/test_train_tokenizer_calls_gpu.py): every conv of the training forward (ResidualUnits unfused) and every data
gradient, the calls per kind, and the premises of its replays (the deepest GEMM within the replay grid's exact depth, the
weight-gradient replay's integer sums below 2^24, the slab plans and defect tiles on 132 SMs)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import synth_data
from tests.test_bench_calls_cpu import N_SM
from tests.test_bench_calls_gpu import REPLAY_GRID, last_cta
from tests.util import README_LAYERS

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_ELU, ACT_LEAKY_RELU, ACT_RELU, ACT_SILU, SHUFFLE_SPACE, SHUFFLE_TIME
from magvit2_pytorch_b200.engine import (Engine, pack_conv, pack_conv_down_space, pack_conv_in_kwpack, pack_feed_forward,
                                         pack_linear_attention)
from magvit2_pytorch_b200.gan import logits_conv_weight, stride2_1x1_dgrad_weight, unshuffle_conv_weight, unshuffle_dgrad_weight
from magvit2_pytorch_b200.train import transposed_pack
from magvit2_pytorch_b200.vgg import adaptive_pool_matrix, fold_avgpool_linear

BF = torch.bfloat16
README_TRAIN_KW = dict(image_size=128, init_dim=64, max_dim=512, codebook_size=1024, layers=README_LAYERS)
CLIPS = 4
# the calls that run on the CUDA-core conv by design: block 0's conv_res (3 input channels) and its stride-2 data gradient
# (12 output channels); neither is a multiple of the wgmma kernels' channel granularity
SIMT_BY_DESIGN = {("discr", "res", 0), ("discr", "dgrad_s2", 0)}


def readme_train_model(device="meta"):
    """The README training model's modules (no weights filled)."""
    with torch.device(device):
        return VideoTokenizer(**README_TRAIN_KW, vgg=synth_data.build_vgg(synth_data.VGG16_CFG, 4096))


def _c(net, role, block, x_shape, pk, kw, kind):
    return dict(net=net, role=role, block=block, x_shape=tuple(x_shape), pk=pk, kw=kw, kind=kind)


def discr_calls(d, B):
    """Every engine conv of one DiscrRunner forward and backward (with the image gradient), in gan.py's order:
    dict(net, role, block, x_shape, pk, kw, kind) with kind the kernel it must run."""
    calls, S = [], d.image_size[0]
    for i, (block, attn) in enumerate(d.blocks):
        n0, n2, cr = block.net[0], block.net[2], block.conv_res
        co, ci = n0.weight.shape[:2]
        down = block.downsample is not None
        So = S // 2 if down else S
        if i == 0:
            calls.append(_c("discr", "net0_kw", i, (B, 1, S, S, 32), pack_conv_in_kwpack(n0.weight[:, :, None], n0.bias),
                            dict(pad=(0, 1, 0), act=ACT_LEAKY_RELU), "slab"))
        else:
            calls.append(_c("discr", "net0", i, (B, 1, S, S, ci), pack_conv(n0.weight, n0.bias, BF), dict(act=ACT_LEAKY_RELU),
                            "slab"))
        if down:
            calls.append(_c("discr", "res", i, (B, 1, S, S, ci), pack_conv(cr.weight, cr.bias, BF),
                            dict(stride=(1, 2, 2), pad=(0, 0, 0), out_spatial=(1, So, So)), "simt" if i == 0 else "tap"))
            calls.append(_c("discr", "net2", i, (B, 1, S, S, co), pack_conv(n2.weight, n2.bias, BF), dict(act=ACT_LEAKY_RELU),
                            "slab"))
            pk = pack_conv(unshuffle_conv_weight(block.downsample[1].weight), block.downsample[1].bias, BF)
            pk.epi_mode = 2
            calls.append(_c("discr", "down", i, (B, 1, S, S, co), pk,
                            dict(stride=(1, 2, 2), pad=(0, 0, 0), out_spatial=(1, So, So), res=True), "tap"))
        else:
            calls.append(_c("discr", "net2", i, (B, 1, S, S, co), pack_conv(n2.weight, n2.bias, BF), dict(act=ACT_LEAKY_RELU),
                            "slab"))
            pk = pack_conv(cr.weight, cr.bias, BF)
            pk.epi_mode = 2
            calls.append(_c("discr", "res_scaled", i, (B, 1, S, S, ci), pk, dict(res=True), "slab"))
        la, ff = attn[0].fn, attn[1].fn
        x = (B, 1, So, So, co)
        inner = la.heads * la.dim_head
        calls += [_c("discr", "q", i, x, pack_conv(la.attn.to_q[0].weight[:, :, None, None, None], None, BF), {}, "slab"),
                  _c("discr", "kv", i, x, pack_conv(la.attn.to_kv[0].weight[:, :, None, None, None], None, BF), {}, "slab"),
                  _c("discr", "out", i, x[:-1] + (inner,), pack_conv(la.attn.to_out[0].weight[:, :, None, None, None], None, BF),
                     dict(res=True), "slab")]
        p = pack_feed_forward(ff, BF)
        calls += [_c("discr", "fc1", i, x, p["fc1"], {}, "slab"),
                  _c("discr", "fc2", i, x[:-1] + (p["fc1"].Co_tc // 2,), p["fc2"], dict(res=True), "slab")]
        # the data gradients of the block's backward (gan.DiscrRunner._block): net2 (3x3), the unshuffle conv (stride 2),
        # net0 (3x3; in block 0 the image gradient) and conv_res (stride 2, or a 1x1 stride-1 conv without downsample)
        calls.append(_dgrad_call("discr", i, n2.weight, (B, 1, S, S, co), "slab"))
        if down:
            calls.append(_s2_call(i, unshuffle_dgrad_weight(block.downsample[1].weight), (B, 1, So, So, co), "slab"))
        calls.append(_dgrad_call("discr", i, n0.weight, (B, 1, S, S, co), "slab"))
        if down:
            calls.append(_s2_call(i, stride2_1x1_dgrad_weight(cr.weight), (B, 1, So, So, co), "simt" if i == 0 else "slab"))
        else:
            calls.append(_dgrad_call("discr", i, cr.weight, (B, 1, S, S, co), "slab"))
        S = So
    tl = d.to_logits
    C_ = tl[0].weight.shape[0]
    x = (B, 1, S, S, C_)
    calls += [_c("discr", "logits_conv", None, x, pack_conv(tl[0].weight, tl[0].bias, BF), dict(act=ACT_LEAKY_RELU), "slab"),
              _c("discr", "logits_lin", None, x, pack_conv(logits_conv_weight(tl[3], C_, d.last_fmap), tl[3].bias, BF),
                 dict(pad=(0, 0, 0), out_spatial=(1, 1, 1)), "tap"),
              _dgrad_call("discr", None, tl[0].weight, x, "slab")]
    return calls


def _dgrad_call(net, block, w, g_shape, kind):
    """TapeRunner._dgrad of a stride-1 conv with weight w (Co, Ci, kh, kw): the transposed conv on g (B, 1, H, W, Co)."""
    kh, kw = w.shape[2:]
    return _c(net, f"dgrad k{kh}{kw}", block, g_shape, transposed_pack(w, (1, kh, kw), BF),
              dict(pad=(0, kh // 2, kw // 2), out_spatial=g_shape[1:4]), kind)


def _s2_call(block, wd, g_shape, kind):
    """DiscrRunner._dgrad_s2: the 1x1 conv C_out -> 4 C_in with the depth-to-space store."""
    return _c("discr", "dgrad_s2", block, g_shape, pack_conv(wd, None, BF, shuffle_q=4), dict(shuffle=SHUFFLE_SPACE), kind)


def vgg_calls(vgg, B, S):
    """Every engine conv of one VggRunner forward and data gradient (vgg.py), as discr_calls."""
    calls, first = [], True
    for m in vgg.features:
        if isinstance(m, torch.nn.Conv2d):
            x = (B, 1, S, S, m.weight.shape[1])
            if first:
                calls.append(_c("vgg", "conv_kw", 0, (B, 1, S, S, 32), pack_conv_in_kwpack(m.weight[:, :, None], m.bias),
                                dict(pad=(0, 1, 0), act=ACT_RELU), "slab"))
            else:
                calls.append(_c("vgg", "conv", None, x, pack_conv(m.weight, m.bias, BF), dict(act=ACT_RELU), "slab"))
            calls.append(_dgrad_call("vgg", 0 if first else None, m.weight, x[:-1] + (m.weight.shape[0],), "slab"))
            first, c_last = False, m.weight.shape[0]
        elif isinstance(m, torch.nn.MaxPool2d):
            S //= 2
    lins = [m for m in vgg.classifier if isinstance(m, torch.nn.Linear)]
    l1, l2 = lins
    oh, ow = vgg.avgpool.output_size
    wf = fold_avgpool_linear(l1.weight, c_last, (S, S), (oh, ow))
    calls += [_c("vgg", "linear1", None, (B, 1, S, S, c_last), pack_conv(wf, l1.bias, BF),
                 dict(pad=(0, 0, 0), out_spatial=(1, 1, 1), act=ACT_RELU), "tap"),
              _c("vgg", "linear1_t", None, (B, 1, 1, 1, l1.weight.shape[0]),
                 pack_conv(wf.permute(2, 3, 1, 0).reshape(S * S * c_last, -1)[:, :, None, None], None, BF), {}, "tap"),
              _c("vgg", "linear2", None, (B, 1, 1, 1, l2.weight.shape[1]), pack_conv(l2.weight[:, :, None, None], l2.bias, BF),
                 dict(act=ACT_RELU), "slab"),
              _c("vgg", "linear2_t", None, (B, 1, 1, 1, l2.weight.shape[0]), pack_conv(l2.weight.t()[:, :, None, None], None, BF),
                 {}, "slab")]
    return calls


def call_key(c):
    """What identifies a call in the table: network, role, input shape, output channels of the GEMM."""
    return (c["net"], c["role"], tuple(c["x_shape"]), c["pk"].Co)


def readme_table():
    """{call_key: (kind, block)} of the README training step's discriminator and VGG calls."""
    m = readme_train_model()
    calls = discr_calls(m.discr, CLIPS) + vgg_calls(m.vgg, CLIPS, 128)
    table = {}
    for c in calls:
        table[call_key(c)] = (c["kind"], c["block"])
    return calls, table


def _n_linear(vgg):
    return sum(isinstance(m, torch.nn.Linear) for m in vgg.classifier)


def discr_counts(d, image_grad):
    """(forward, backward) calls per kind of one DiscrRunner: per block net0 (the kw-packed ingest in block 0), conv_res,
    net2 and the unshuffle conv (down-sampling blocks) or the scaled conv_res, q / kv / out and fc1 / fc2 with two
    rmsnorms; to_logits' conv and Linear.  Backward: per block the net2 dgrad, the unshuffle conv's stride-2 dgrad, and
    -- unless block 0 without the image gradient -- the net0 dgrad and conv_res's (stride-2 or 1x1) dgrad; to_logits'
    3x3 dgrad."""
    fwd = dict(conv=2, rmsnorm=0, ingest=1)
    bwd = dict(dgrad=1, dgrad_s2=0)
    for i, (block, _) in enumerate(d.blocks):
        down = block.downsample is not None
        fwd["conv"] += (4 if down else 3) + 5
        fwd["rmsnorm"] += 2
        bwd["dgrad"] += 1
        bwd["dgrad_s2"] += down
        if i > 0 or image_grad:
            bwd["dgrad"] += 1 + (not down)
            bwd["dgrad_s2"] += down
    return fwd, bwd


def vgg_counts(vgg):
    """(forward, backward) calls per kind of one VggRunner: every 3x3 conv and every Linear a conv, one pool per
    MaxPool2d, the kw-packed ingest; backward: a dgrad per conv, a pool backward per pool, a transposed conv per Linear."""
    n_conv = sum(isinstance(m, torch.nn.Conv2d) for m in vgg.features)
    n_pool = sum(isinstance(m, torch.nn.MaxPool2d) for m in vgg.features)
    n_lin = _n_linear(vgg)
    return dict(conv=n_conv + n_lin, maxpool=n_pool, ingest=1), dict(dgrad=n_conv, maxpool_bwd=n_pool, linear_t=n_lin)


def step_counts(m):
    """Calls per (network, kind) of the generator step and the discriminator step (tests/test_train_calls_gpu.py): the
    generator step runs the discriminator forward and backward with the image gradient, the VGG forward on the real and
    the reconstructed frames, the VGG's data gradient and one mse; the discriminator step two discriminator forwards and
    backwards without an image gradient."""
    fwd_g, bwd_g = discr_counts(m.discr, True)
    fwd_d, bwd_d = discr_counts(m.discr, False)
    fwd_v, bwd_v = vgg_counts(m.vgg)
    gen = {("discr", k): v for k, v in {**fwd_g, **bwd_g}.items()}
    gen.update({("vgg", k): 2 * v for k, v in fwd_v.items()})
    gen.update({("vgg", k): v for k, v in bwd_v.items()})
    gen[("vgg", "mse")] = 1
    dis = {("discr", k): 2 * v for k, v in {**fwd_d, **bwd_d}.items()}
    return gen, dis


# ------------------------------------------------------------------------------------------------------------------
def _engine():
    eng = Engine(None)
    eng.dtype = BF
    return eng


def test_readme_train_call_kernels():
    """Every discriminator and VGG call of the README training step runs the kernel of the table."""
    eng = _engine()
    calls, table = readme_table()
    got = {}
    for c in calls:
        kw = dict(c["kw"])
        res = kw.pop("res", False)
        ta = eng._tc_args(c["x_shape"], c["pk"], res=torch.empty(1) if res else None, **kw)
        got[call_key(c)] = eng.conv_kernel(ta, c["pk"])
    assert got == {k: v[0] for k, v in table.items()}
    simt = {(c["net"], c["role"], c["block"]) for c in calls if c["kind"] == "simt"}
    assert simt == SIMT_BY_DESIGN, simt
    # the shapes the issue of these calls is about: depth-8192 tap calls, 4096-deep 1x1 calls, 3-channel image dgrads, 3x3
    # convs on the 4 x 4 map
    depth = {call_key(c): math.prod(c["pk"].k_tc) * c["pk"].Ci_tc for c in calls}
    assert {k[:2] for k, K in depth.items() if K == 8192} == {("discr", "logits_lin"), ("vgg", "linear1")}
    assert {k[:2] for k, K in depth.items() if K == 4096} >= {("vgg", "linear2"), ("vgg", "linear2_t"), ("vgg", "linear1_t")}
    assert {(k[0], k[2][2]) for k in table if k[1] == "dgrad k33" and k[3] == 3} == {("discr", 128), ("vgg", 128)}
    assert {k[1] for k in table if k[0] == "discr" and k[2][2] == 4 and k[1] != "logits_lin"} >= {
        "net0", "net2", "logits_conv", "dgrad k33"}


def test_readme_train_call_counts():
    """The call-count formulas on the README modules: six discriminator blocks (five down-sampling) plus to_logits;
    VGG16's 13 convs, 5 pools and 2 Linears."""
    m = readme_train_model()
    d, vgg = m.discr, m.vgg
    assert len(d.blocks) == 6 and sum(b.downsample is not None for b, _ in d.blocks) == 5 and d.last_fmap == (4, 4)
    assert vgg_counts(vgg) == (dict(conv=15, maxpool=5, ingest=1), dict(dgrad=13, maxpool_bwd=5, linear_t=2))
    # forward: 5 x (4 + 5) + (3 + 5) + 2 convs, 12 rmsnorms; backward with the image gradient: 6 net2 + 6 net0 + 1 conv_res
    # (1x1, block 5) + to_logits dgrads, 5 unshuffle + 5 conv_res stride-2 dgrads; without: block 0's net0 / conv_res less
    assert discr_counts(d, True) == (dict(conv=55, rmsnorm=12, ingest=1), dict(dgrad=14, dgrad_s2=10))
    assert discr_counts(d, False) == (dict(conv=55, rmsnorm=12, ingest=1), dict(dgrad=13, dgrad_s2=9))
    calls, table = readme_table()
    n_fwd = sum(c["net"] == "discr" and not c["role"].startswith("dgrad") for c in calls)
    n_bwd = sum(c["net"] == "discr" and c["role"].startswith("dgrad") for c in calls)
    assert (n_fwd, n_bwd) == (55, 24)
    gen, dis = step_counts(m)
    assert gen[("vgg", "conv")] == 30 and gen[("vgg", "dgrad")] == 13 and dis[("discr", "conv")] == 110


def test_replay_grid_is_exact_at_every_depth():
    (nx, ex), (nw, ew), (nb, eb) = REPLAY_GRID["x"], REPLAY_GRID["w"], REPLAY_GRID["b"]
    calls, _ = readme_table()
    ks = sorted({math.prod(c["pk"].k_tc) * c["pk"].Ci_tc for c in calls if c["kind"] != "simt"})
    assert max(ks) == 8192, ks
    # the arithmetic: products are multiples of 2^-(ex + ew) of magnitude <= nx nw 2^-(ex + ew) = 0.25; the bias a multiple of
    # 2^-eb, eb <= ex + ew; every partial sum (all products of one sign at their largest, plus the bias) stays below
    # 2^(22 - ex - ew) = 2^14, so it has at most 22 significant bits
    m_ = ex + ew
    assert eb <= m_ and nx * nw * 2.0 ** -m_ == 0.25
    for K in ks:
        worst = K * nx * nw * 2.0 ** -m_ + nb * 2.0 ** -eb
        assert worst < 2.0 ** (22 - m_), (K, worst)
    assert 8192 * 0.25 == 2.0 ** 11
    # fp32 sums, in three shuffled orders, of the worst case and of random grid operands equal the float64 sums
    rng = np.random.default_rng(8192)
    for K in (8192, 4096, 9 * 512, 9 * 64):
        assert K in ks, K
        worst = np.full(K + 1, nx * nw * 2.0 ** -m_)
        worst[-1] = nb * 2.0 ** -eb
        rand = np.append(rng.integers(-nx, nx + 1, K) * rng.integers(-nw, nw + 1, K) * 2.0 ** -m_,
                         rng.integers(-nb, nb + 1) * 2.0 ** -eb)
        for terms in (worst, -worst, rand):
            exact = terms.sum()
            for _ in range(3):
                order = rng.permutation(K + 1)
                part = np.cumsum(terms[order].astype(np.float32), dtype=np.float32)
                assert part[-1] == exact and np.array_equal(part.astype(np.float64), np.cumsum(terms[order]))


@pytest.mark.parametrize("fmap", [(4, 4), (7, 7), (3, 5)])
def test_fold_error_allowance(fmap):
    """The allowance the GPU test adds for the VGG's first Linear (the average pool folded into its weights in fp32, then
    rounded to bf16): |bf16(fp32(w_fold)) - w_fold| <= (2^-8 + 2^-23) |w_fold| per weight, on bf16 Linear weights."""
    g = torch.Generator().manual_seed(sum(fmap))
    w = (torch.randn(64, 8 * 49, generator=g) * 0.05).to(BF)
    wf64 = torch.einsum("ocij,iy,jx->ocyx", w.double().reshape(64, 8, 7, 7),
                        *(adaptive_pool_matrix(n, 7) for n in fmap))
    wf = fold_avgpool_linear(w, 8, fmap, (7, 7)).to(BF).double()
    assert ((wf - wf64).abs() <= (2.0 ** -8 + 2.0 ** -23) * wf64.abs()).all()


# ------------------------------------------------------------------------------------------------------------------
# the tokenizer's own calls (tests/test_train_tokenizer_calls_gpu.py)
# ------------------------------------------------------------------------------------------------------------------
FRAMES = 17
# the tokenizer call that runs on the CUDA-core conv by design: conv_out's data gradient, a transposed conv with 3 input
# channels (the reconstruction's), below the wgmma kernels' channel granularity
TOK_SIMT_BY_DESIGN = {("tok", "dgrad k333", "conv_out")}


def _tok_dgrad(block, w, k, g_shape, kind):
    """TapeRunner._dgrad of a stride-1 causal conv with weight w and kernel k: the transposed conv on g (B, T, H, W, Co)."""
    return _c("tok", f"dgrad k{''.join(map(str, k))}", block, g_shape, transposed_pack(w, k, BF),
              dict(pad=(0, k[1] // 2, k[2] // 2), out_spatial=g_shape[1:4]), kind)


def _attn_calls(calls, key, mod, st, x):
    """The convs of an attention-type stage: its projections, then the feed-forward's fc1 (GEGLU) and fc2."""
    time_axis = st.kind == "attend_time"
    if st.kind == "linear_attend_space":
        p = pack_linear_attention(mod[0].fn, BF)
        inner = p["heads"] * p["dim_head"]
        calls += [_c("tok", "q", key, x, p["q"], {}, "slab"), _c("tok", "kv", key, x, p["kv"], {}, "slab"),
                  _c("tok", "attn_out", key, x[:-1] + (inner,), p["out"], dict(res=True), "slab")]
        ff = mod[1].fn
    else:
        at = mod[0].fn.fn if time_axis else mod[0].fn
        inner = at.heads * at.dim_head
        calls += [_c("tok", "qkv", key, x, pack_conv(at.to_qkv[0].weight[:, :, None, None, None], None, BF), {}, "slab"),
                  _c("tok", "attn_out", key, x[:-1] + (inner,),
                     pack_conv(at.to_out[1].weight[:, :, None, None, None], None, BF), dict(res=True), "slab")]
        ff = mod[1].fn.fn if time_axis else mod[1].fn
    p = pack_feed_forward(ff, BF)
    calls += [_c("tok", "fc1", key, x, p["fc1"], {}, "slab"),
              _c("tok", "fc2", key, x[:-1] + (p["fc1"].Co_tc // 2,), p["fc2"], dict(res=True), "slab")]


def tokenizer_calls(m, B, frames=FRAMES, size=128):
    """Every engine conv of one TrainRunner forward and backward of the tokenizer (train.py), in the order of the forward,
    then the data gradients: dict(net, role, block, x_shape, pk, kw, kind) as discr_calls.  The ResidualUnits run unfused
    (conv3 with ELU, conv1 with ELU); the backward runs two data gradients per ResidualUnit and conv_out's."""
    T, S = frames + m.time_padding, size
    cin = m.conv_in.conv
    pin = pack_conv_in_kwpack(cin.weight, cin.bias)
    kt, kh = pin.k_tc[:2]
    calls = [_c("tok", "conv_in_kw", "conv_in", (B, T, S, S, pin.Ci_tc), pin, dict(pad=(kt - 1, kh // 2, 0)), "slab")]
    dgrads = []

    def residual(key, mod, st, x):
        for j, ru in enumerate(list(mod) if st.nested else [mod]):
            seq = ru.fn
            c3, c1 = seq[0].conv, seq[2]
            k3 = tuple(c3.weight.shape[2:])
            calls.append(_c("tok", "conv3", f"{key}.{j}", x, pack_conv(c3.weight, c3.bias, BF), dict(act=ACT_ELU), "slab"))
            calls.append(_c("tok", "conv1", f"{key}.{j}", x, pack_conv(c1.weight, c1.bias, BF), dict(act=ACT_ELU), "slab"))
            dgrads.append(_tok_dgrad(f"{key}.{j}", c1.weight, (1, 1, 1), x, "slab"))
            dgrads.append(_tok_dgrad(f"{key}.{j}", c3.weight, k3, x, "slab"))

    C_ = cin.weight.shape[0]
    for i, st in enumerate(m.stages):
        mod, key, x = m.encoder_layers[i], f"enc{i}", (B, T, S, S, C_)
        if st.kind == "residual":
            residual(key, mod, st, x)
        elif st.kind == "compress_space":
            pk = pack_conv(mod.conv.weight, mod.conv.bias, BF)
            pack_conv_down_space(pk, mod.conv.weight)
            S //= 2
            calls.append(_c("tok", "down_space", key, x, pk, dict(stride=(1, 2, 2), pad=(0, 1, 1), out_spatial=(T, S, S)),
                            "down"))
            C_ = pk.Co
        elif st.kind == "compress_time":
            pk = pack_conv(mod.conv.weight, mod.conv.bias, BF, k=(3, 1, 1))
            T //= 2
            calls.append(_c("tok", "down_time", key, x, pk, dict(stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=(T, S, S)),
                            "slab"))
            C_ = pk.Co
        else:
            _attn_calls(calls, key, mod, st, x)
    for j, st in enumerate(reversed(m.stages)):
        mod, key, x = m.decoder_layers[j], f"dec{j}", (B, T, S, S, C_)
        if st.kind == "residual":
            residual(key, mod, st, x)
        elif st.kind == "compress_space":
            pk = pack_conv(mod.net[0].weight, mod.net[0].bias, BF, shuffle_q=4)
            calls.append(_c("tok", "up_space", key, x, pk, dict(act=ACT_SILU, shuffle=SHUFFLE_SPACE), "slab"))
            S, C_ = 2 * S, pk.Co // 4
        elif st.kind == "compress_time":
            pk = pack_conv(mod.net[0].weight, mod.net[0].bias, BF, k=(1, 1, 1), shuffle_q=2)
            calls.append(_c("tok", "up_time", key, x, pk, dict(act=ACT_SILU, shuffle=SHUFFLE_TIME), "slab"))
            T, C_ = 2 * T, pk.Co // 2
        else:
            _attn_calls(calls, key, mod, st, x)
    cout = m.conv_out.conv
    kout, tp = tuple(cout.weight.shape[2:]), m.time_padding
    x = (B, T, S, S, C_)
    calls.append(_c("tok", "conv_out", "conv_out", x, pack_conv(cout.weight, cout.bias, BF),
                    dict(pad=(kout[0] - 1 - tp, kout[1] // 2, kout[2] // 2), out_spatial=(T - tp, S, S), out_cf=True), "slab"))
    dgrads.append(_tok_dgrad("conv_out", cout.weight, kout, x[:-1] + (cout.weight.shape[0],), "simt"))
    return calls + dgrads


def tokenizer_table(B=CLIPS):
    """(calls, {call_key: (kind, block)}, model) of the README training step's tokenizer calls."""
    m = readme_train_model()
    calls = tokenizer_calls(m, B)
    return calls, {call_key(c): (c["kind"], c["block"]) for c in calls}, m


def _n_residual_units(m):
    return sum(st.count for st in m.stages if st.kind == "residual")


def tokenizer_counts(m):
    """Calls per kind of the tokenizer in one generator step (TrainRunner forward, backward and the adaptive weight's two
    last_layer_weight_grad calls): per ResidualUnit two convs, one squeeze_excite_residual, two data gradients and two
    _conv_bwd; per attention-type stage (each side) the projections (3 for the linear attention, 2 otherwise), fc1, fc2 and
    two rmsnorms; one conv per down- or up-sampler and one _conv_bwd per down-sampler (its weight and data gradient); conv_in
    and conv_out, conv_in's _conv_bwd (weights only), conv_out's data gradient and three _conv_bwd through
    _conv_bwd_padmode (the backward, and weights only for each last_layer_weight_grad); one quantize_cl and one batch-entropy
    start / finish."""
    n_ru = 2 * _n_residual_units(m)
    n = dict(conv=2 + 2 * n_ru, se=n_ru, rmsnorm=0, dgrad=2 * n_ru + 1, conv_bwd=2 * n_ru + 1 + 3, padmode=3,
             quantize=1, entropy=1)
    for st in m.stages:
        if st.kind in ("compress_space", "compress_time"):
            n["conv"] += 2
            n["conv_bwd"] += 1
        elif st.kind in ("attend_space", "attend_time", "linear_attend_space"):
            n["conv"] += 2 * ((3 if st.kind == "linear_attend_space" else 2) + 2)
            n["rmsnorm"] += 4
    return n


def test_readme_train_tokenizer_call_kernels():
    """Every tokenizer conv and data gradient of the README training step runs the kernel of the table: the slab kernel,
    its down-space flavour for the three SpatialDownsample2x, and the CUDA-core conv only for conv_out's data gradient."""
    eng = _engine()
    calls, table, _ = tokenizer_table()
    got = {}
    for c in calls:
        kw = dict(c["kw"])
        res = kw.pop("res", False)
        ta = eng._tc_args(c["x_shape"], c["pk"], res=torch.empty(1) if res else None, **kw)
        got[call_key(c)] = eng.conv_kernel(ta, c["pk"])
    assert got == {k: v[0] for k, v in table.items()}
    assert {(c["net"], c["role"], c["block"]) for c in calls if c["kind"] == "simt"} == TOK_SIMT_BY_DESIGN
    assert {c["block"] for c in calls if c["kind"] == "down"} == {"enc1", "enc3", "enc6"}


def test_readme_train_tokenizer_call_counts():
    """The count formulas on the README modules: 11 ResidualUnits per side, three space and two time samplers, one
    linear, one space and one time attention stage."""
    calls, table, m = tokenizer_table()
    assert _n_residual_units(m) == 11 and m.time_padding == 3
    n = tokenizer_counts(m)
    assert n == dict(conv=82, se=22, rmsnorm=12, dgrad=45, conv_bwd=53, padmode=3, quantize=1, entropy=1), n
    assert sum(not c["role"].startswith("dgrad") for c in calls) == n["conv"]
    assert sum(c["role"].startswith("dgrad") for c in calls) == n["dgrad"]


def test_tokenizer_replay_premises():
    """The exact replays of tests/test_train_tokenizer_calls_gpu.py:
      * the deepest wgmma GEMM is the 512-channel 3x3x3 conv and its data gradient, K = 13824, within the depth up to which
        tests/test_bench_calls_cpu.py shows REPLAY_GRID exact (27 x 1024);
      * the weight-gradient replays take operands in {-1, 0, 1}: at the deepest summation, 4 clips x 20 frames x 128^2
        positions, every partial sum is an integer of magnitude below 2^24, exact in fp32 in any order;
      * mv2_tc_slab_plan on 132 SMs: the 64-channel 128^2 unfused ResidualUnit convs and their data gradients plan 5120 tiles
        on a grid of 132 (39 per CTA, rounded up), the 512-channel 16^2 calls at 5 frames 160 tiles on 132 CTAs, and every
        slab call plans more tiles than CTAs;
      * the schedule's last tile of every slab call has a predecessor on its CTA whose output region does not overlap it,
        so a previous tile's accumulators left in place are visible there."""
    calls, _, _ = tokenizer_table()
    ks = {math.prod(c["pk"].k_tc) * c["pk"].Ci_tc for c in calls if c["kind"] != "simt"}
    assert max(ks) == 27 * 512 <= 27 * 1024
    assert {c["role"] for c in calls if c["kind"] != "simt" and math.prod(c["pk"].k_tc) * c["pk"].Ci_tc == max(ks)} == {
        "conv3", "dgrad k333"}
    assert CLIPS * (FRAMES + 3) * 128 * 128 == 1310720 < 2 ** 24
    eng, lib = _engine(), Engine(None).lib
    out = (C.c_int32 * 6)()
    n_slab = 0
    for c in calls:
        if c["kind"] != "slab":
            continue
        kw = dict(c["kw"])
        res = kw.pop("res", False)
        ta = eng._tc_args(c["x_shape"], c["pk"], res=torch.empty(1) if res else None, **kw)
        ta.x = ta.w = ta.y = 1
        assert lib.mv2_tc_slab_plan(C.byref(ta), N_SM, out) == 0, lib.mv2_last_error()
        mw, bn, total, grid = out[0], out[1], out[3], out[4]
        assert total > grid == N_SM, (call_key(c), total, grid)
        if c["role"] in ("conv3", "conv1", "dgrad k333", "dgrad k111") and c["x_shape"][1:] == (20, 128, 128, 64):
            assert (total, grid, -(-total // grid)) == (5120, 132, 39), call_key(c)
        if c["x_shape"][1:4] == (5, 16, 16) and c["pk"].Co_tc == 512:
            assert (total, grid) == (160, 132), call_key(c)
        tiles, k = [], 0
        while True:
            assert lib.mv2_tc_slab_tile(C.byref(ta), N_SM, last_cta(total, grid), k, out) == 0
            if out[0] < 0:
                break
            tiles.append(tuple(out))
            k += 1
        assert len(tiles) >= 2 and tiles[-1][0] == total - 1, (call_key(c), tiles)
        (_, b0, t0, h0, w0, n0), (_, b1, t1, h1, w1, n1) = tiles[-2:]
        assert not (b0 == b1 and t0 == t1 and abs(h0 - h1) < 16 and abs(w0 - w1) < 8 * mw and abs(n0 - n1) < bn), (
            call_key(c), tiles[-2:])
        n_slab += 1
    assert n_slab == sum(c["kind"] == "slab" for c in calls)
