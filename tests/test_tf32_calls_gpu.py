"""The TF32 conv kernels, one Engine.conv call at a time, against float64 at their edges: every flavour the TF32 slab
kernel has (plain, residual, GEGLU, SpatialDownsample2x, the stride-2 TimeDownsample2x, the depth-to-space / depth-to-time
stores, the channels-first conv_out store) and the tap-wise kernel, with ragged N tiles, frames whose H and W are not
tile multiples, causal leading frames and the history operand of a streamed clip.

Operand rounding (DESIGN.md): the tensor core reads each fp32 operand as TF32, its top 19 bits, so the float64 reference
runs on operands with the low 13 mantissa bits cleared.  The products of such operands are exact in fp32; what remains is
the fp32 accumulation order, bounded by K * 2^-23 * sum |a b| (K products, one unit of the last place per addition), and the
activations' approximations (2^-21 relative, 2^-22 absolute).  test_operands_are_truncated_not_rounded checks the rounding
model itself on sums that tell truncation and rounding apart."""
import pytest
import torch
import torch.nn.functional as F

from magvit2_pytorch_b200._lib import ACT_ELU, ACT_NONE, ACT_SILU, SHUFFLE_SPACE, SHUFFLE_TIME
from magvit2_pytorch_b200.engine import Engine, StreamState, pack_conv, pack_conv_down_space, pack_ff

pytestmark = pytest.mark.gpu


def tf32_trunc(t):
    """fp32 -> the TF32 value the tensor core reads (low 13 mantissa bits cleared), as float64."""
    i = t.float().contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32).double()


@pytest.fixture(scope="module")
def eng():
    e = Engine(None)
    e.bind(torch.zeros(1, device="cuda"), "test")
    e.tf32 = True
    return e


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).float()


def _ref(x, w, b, stride, pad, act=ACT_NONE, res=None, rs=1.0):
    """float64 conv of channels-last x (B, T, H, W, Ci) with torch weight w (Co, Ci, kt, kh, kw), leading pad (pt, ph, pw)
    (trailing spatial pad the same, as a symmetric 'same' conv), on TF32 operands -> (y, bound)."""
    xt, wt = tf32_trunc(x).permute(0, 4, 1, 2, 3), tf32_trunc(w)
    pt, ph, pw = pad
    xp = F.pad(xt, (pw, pw, ph, ph, pt, 0))
    z = F.conv3d(xp, wt, None, stride)
    S = F.conv3d(xp.abs(), wt.abs(), None, stride)
    K = w[0].numel()
    if b is not None:
        z = z + b.double()[None, :, None, None, None]
        S = S + b.double().abs()[None, :, None, None, None]
    bound = K * 2.0 ** -23 * S
    if act == ACT_ELU:
        y = F.elu(z)
        bound = bound + 2.0 ** -21 * y.abs() + 2.0 ** -22
    elif act == ACT_SILU:
        y = F.silu(z)
        bound = bound + 2.0 ** -21 * (y.abs() + z.abs()) + 2.0 ** -22
    else:
        y = z
    y, bound = y.permute(0, 2, 3, 4, 1), bound.permute(0, 2, 3, 4, 1)
    if res is not None:
        y = (y + res.double()) * rs
        bound = (bound + 2.0 ** -24 * y.abs()) * rs
    return y, bound + 2.0 ** -24 * y.abs()


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    assert torch.isfinite(got).all(), what
    excess = (err - bound).max().item()
    assert excess <= 0, (what, excess, err.max().item())


def _conv_case(eng, Ci, Co, k, B=2, T=4, H=20, W=19, act=ACT_ELU, res=False, tap=False, hist=False):
    torch.manual_seed(Ci * 7 + Co)
    w, b = _rand(Co, Ci, *k, scale=Ci ** -0.5), _rand(Co, scale=0.1)
    pk = pack_conv(w, b, torch.float32, tc=True)
    x = _rand(B, T, H, W, Ci)
    r = _rand(B, T, H, W, Co) if res else None
    eng.tc_variant = "tap" if tap else "auto"
    eng.conv_log = []
    try:
        if hist:      # two chunks of one streamed clip: the second reads its leading frames from the history operand
            ss = StreamState()
            y = torch.cat([eng.conv(x[:, :2].contiguous(), pk, act=act, ss=ss.sub("c")),
                           eng.conv(x[:, 2:].contiguous(), pk, act=act, ss=ss.sub("c"))], 1)
        else:
            y = eng.conv(x, pk, act=act, res=r)
        kinds = {rec["kind"] for rec in eng.conv_log}
    finally:
        eng.tc_variant, eng.conv_log = "auto", None
    ref, bound = _ref(x, w, b, (1, 1, 1), (k[0] - 1, k[1] // 2, k[2] // 2), act, r)
    return y, ref, bound, kinds


@pytest.mark.parametrize("Ci,Co,k,kw", [
    (64, 64, (3, 3, 3), {}),                       # the causal 3x3x3 conv of a ResidualUnit (unfused in TF32)
    (128, 128, (3, 3, 3), dict(H=17, W=33)),       # H, W not tile multiples
    (32, 64, (1, 1, 1), dict(res=True, act=ACT_NONE)),   # Linear with the residual epilogue
    (64, 2080, (1, 1, 1), dict(act=ACT_NONE, H=8, W=8)),   # 128-column N tiles with a ragged last one
    (16, 96, (1, 1, 1), dict(act=ACT_SILU)),       # 64-byte K rows
    (64, 64, (3, 3, 3), dict(hist=True)),           # the history operand
    (64, 64, (3, 3, 3), dict(tap=True)),            # tap-wise kernel
    (24, 40, (3, 3, 3), dict(tap=True)),            # tap-wise, 32-byte K rows, ragged N
])
def test_conv_vs_float64(eng, Ci, Co, k, kw):
    y, ref, bound, kinds = _conv_case(eng, Ci, Co, k, **kw)
    assert kinds == {"tap" if kw.get("tap") else "slab"}, kinds
    _check(y, ref, bound, (Ci, Co, k, kw))


def test_geglu_vs_float64(eng):
    torch.manual_seed(1)
    C_, I = 64, 96
    w1, b1, w2, b2 = _rand(2 * I, C_, 1, 1, 1, scale=0.125), _rand(2 * I, scale=0.1), _rand(C_, I, 1, 1, 1), _rand(C_)
    fc1, _ = pack_ff(w1, b1, w2, b2, torch.float32, tc=True)
    x = _rand(2, 3, 9, 10, C_)
    g = eng.conv(x, fc1)
    z, S = _ref(x, w1, b1, (1, 1, 1), (0, 0, 0))
    h = z[..., :I] * F.gelu(z[..., I:])
    dz = S[..., :I] * F.gelu(z[..., I:]).abs() + S[..., I:] * (z[..., :I].abs() * 1.2)
    assert g.shape[-1] == fc1.Co_tc // 2 and (g[..., I:] == 0).all()      # hidden width padded to 64 with zeros
    _check(g[..., :I], h, dz + 2.0 ** -20 * h.abs() + 2.0 ** -21, "geglu")


def test_strided_and_shuffled_vs_float64(eng):
    torch.manual_seed(2)
    # SpatialDownsample2x on the down-space flavour
    w, b = _rand(128, 64, 3, 3, scale=0.04), _rand(128, scale=0.1)
    pk = pack_conv(w, b, torch.float32, tc=True)
    pack_conv_down_space(pk, w)
    assert pk.w_down is not None
    x = _rand(2, 3, 18, 22, 64)
    eng.conv_log = []
    y = eng.conv(x, pk, stride=(1, 2, 2), pad=(0, 1, 1), out_spatial=(3, 9, 11))
    assert eng.conv_log[-1]["down_space"]
    ref, bound = _ref(x, w[:, :, None], b, (1, 2, 2), (0, 1, 1))
    _check(y, ref[:, :, :9, :11], bound[:, :, :9, :11], "space down")
    # TimeDownsample2x: stride 2 along t, causal pad 2
    w, b = _rand(64, 64, 3, scale=0.07), _rand(64, scale=0.1)
    pk = pack_conv(w, b, torch.float32, k=(3, 1, 1), tc=True)
    x = _rand(2, 5, 12, 12, 64)
    y = eng.conv(x, pk, stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=(3, 12, 12))
    assert eng.conv_log[-1]["kind"] == "slab"
    ref, bound = _ref(x, w[:, :, :, None, None], b, (2, 1, 1), (2, 0, 0))
    _check(y, ref, bound, "time down")
    # depth-to-space (SpatialUpsample2x) and depth-to-time (TimeUpsample2x) stores
    x = _rand(2, 3, 10, 12, 64)
    for q, shuffle in ((4, SHUFFLE_SPACE), (2, SHUFFLE_TIME)):
        w, b = _rand(q * 32, 64, 1, 1, 1, scale=0.125), _rand(q * 32, scale=0.1)
        pk = pack_conv(w, b, torch.float32, k=(1, 1, 1), shuffle_q=q, tc=True)
        y = eng.conv(x, pk, act=ACT_SILU, shuffle=shuffle)
        assert eng.conv_log[-1]["kind"] == "slab"
        ref, bound = _ref(x, w, b, (1, 1, 1), (0, 0, 0), ACT_SILU)       # channels (c, q) as the reference orders them
        B, T, H, W, _ = ref.shape
        if shuffle == SHUFFLE_SPACE:
            arr = lambda t: t.reshape(B, T, H, W, 32, 2, 2).permute(0, 1, 2, 5, 3, 6, 4).reshape(B, T, 2 * H, 2 * W, 32)  # noqa: E731
        else:
            arr = lambda t: t.reshape(B, T, H, W, 32, 2).permute(0, 1, 5, 2, 3, 4).reshape(B, 2 * T, H, W, 32)  # noqa: E731
        _check(y, arr(ref), arr(bound), f"shuffle {shuffle}")
    eng.conv_log = None


def test_channels_first_conv_out_vs_float64(eng):
    torch.manual_seed(3)
    w, b = _rand(3, 64, 3, 3, 3, scale=0.04), _rand(3, scale=0.1)
    pk = pack_conv(w, b, torch.float32, tc=True)
    x = _rand(2, 5, 20, 18, 64)
    assert eng.conv_cf_supported(x, pk, (2, 1, 1), (5, 20, 18))
    y = eng.conv(x, pk, out_cf=True)
    ref, bound = _ref(x, w, b, (1, 1, 1), (2, 1, 1))
    _check(y.permute(0, 2, 3, 4, 1), ref, bound, "conv_out")


@pytest.mark.parametrize("tap", [False, True])
def test_operands_are_truncated_not_rounded(eng, tap):
    """x = 1 + 2^-11 + 2^-12 and w = 1 + 2^-11 + 2^-12: TF32 keeps 10 mantissa bits, so truncation reads 1 and rounding to
    nearest 1 + 2^-10.  Over 32 products the two readings differ by 0.0625, far above the fp32 accumulation bound."""
    v = 1.0 + 2.0 ** -11 + 2.0 ** -12
    x = torch.full((1, 1, 8, 8, 32), v, device="cuda")
    w = torch.full((32, 32, 1, 1, 1), v, device="cuda")
    pk = pack_conv(w, None, torch.float32, tc=True)
    eng.tc_variant = "tap" if tap else "auto"
    try:
        y = eng.conv(x, pk)
    finally:
        eng.tc_variant = "auto"
    assert (y - 32.0).abs().max().item() <= 32 * 32 * 2.0 ** -23, y.flatten()[:4]
