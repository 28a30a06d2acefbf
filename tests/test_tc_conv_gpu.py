"""wgmma implicit-GEMM convolution, shape by shape, through the engine's conv() entry (C ABI underneath), against
(a) the CPU oracle's building blocks (oracle/restated.py: plain torch fp32 functional ops on the same bf16-representable
inputs and weights) and (b) the library's own CUDA-core kernel on identical bf16 inputs (both accumulate in fp32)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R

from magvit2_pytorch_b200 import VideoTokenizer
from magvit2_pytorch_b200._lib import ACT_ELU, ACT_NONE, ACT_SILU, SHUFFLE_NONE, SHUFFLE_SPACE, SHUFFLE_TIME
from magvit2_pytorch_b200.engine import Engine, pack_conv

pytestmark = pytest.mark.gpu

# (name, weight shape (Co,Ci,*k), k3, x shape (B,T,H,W), conv kwargs, shuffle_q)
CASES = [
    ("res3x3x3_c64", (64, 64, 3, 3, 3), None, (1, 3, 32, 32), dict(act=ACT_ELU), 1),
    ("res3x3x3_c128", (128, 128, 3, 3, 3), None, (2, 4, 16, 16), dict(act=ACT_ELU), 1),
    ("res3x3x3_c256", (256, 256, 3, 3, 3), None, (1, 3, 8, 16), dict(), 1),
    ("res3x3x3_c512_2ntiles", (512, 512, 3, 3, 3), None, (1, 2, 8, 8), dict(act=ACT_ELU), 1),
    ("res3x3x3_wide_w128", (64, 64, 3, 3, 3), None, (1, 2, 4, 128), dict(), 1),
    ("res3x3x3_ragged", (64, 64, 3, 3, 3), None, (1, 3, 12, 24), dict(act=ACT_ELU), 1),
    ("pointwise_c64", (64, 64, 1, 1, 1), None, (2, 3, 16, 16), dict(act=ACT_ELU), 1),
    ("linear_512_768", (768, 512, 1, 1, 1), None, (1, 2, 16, 16), dict(), 1),
    ("ff1_ragged_n_256_1364", (1364, 256, 1, 1, 1), None, (1, 2, 8, 8), dict(), 1),
    ("residual_add", (256, 128, 1, 1, 1), None, (1, 2, 16, 16), dict(res=True), 1),
    ("conv_out_co3", (3, 64, 3, 3, 3), None, (1, 3, 16, 32), dict(), 1),
    ("down_space", (128, 64, 3, 3), None, (2, 3, 32, 32), dict(stride=(1, 2, 2), pad=(0, 1, 1), down="space"), 1),
    ("down_time", (512, 512, 3), (3, 1, 1), (1, 8, 8, 8), dict(stride=(2, 1, 1), pad=(2, 0, 0), down="time"), 1),
    ("down_time_oddT", (64, 64, 3), (3, 1, 1), (1, 5, 8, 16), dict(stride=(2, 1, 1), pad=(2, 0, 0), down="time"), 1),
    ("up_space", (256, 128, 1, 1), None, (1, 3, 16, 16), dict(act=ACT_SILU, shuffle=SHUFFLE_SPACE), 4),
    ("up_time", (1024, 512, 1), (1, 1, 1), (1, 3, 8, 8), dict(act=ACT_SILU, shuffle=SHUFFLE_TIME), 2),
    ("bk32_c32", (32, 32, 3, 3, 3), None, (1, 3, 8, 8), dict(act=ACT_ELU), 1),
    ("bk16_c16", (16, 16, 3, 3, 3), None, (1, 3, 16, 16), dict(act=ACT_ELU), 1),
    ("bk16_c48_tinyspatial", (64, 48, 3, 3, 3), None, (2, 3, 4, 4), dict(), 1),
    ("up_space_small_cy16", (64, 32, 1, 1), None, (1, 2, 8, 8), dict(act=ACT_SILU, shuffle=SHUFFLE_SPACE), 4),
]


def _oracle_conv(w, bias, x_cl, k3, kw, res=None):
    """fp32 CPU reference of one conv() call from the oracle's building blocks.  x_cl: (B,T,H,W,Ci) bf16 on the device;
    w: torch-layout fp32 weight (rounded through bf16 here, as the engine packs it); returns channels-last fp32 (CPU)."""
    x = x_cl.float().cpu().permute(0, 4, 1, 2, 3).contiguous()
    wb = w.detach().to(torch.bfloat16).float().cpu()
    b = bias.detach().float().cpu()
    act, shuffle, stride = kw.get("act", ACT_NONE), kw.get("shuffle", SHUFFLE_NONE), kw.get("stride", (1, 1, 1))
    if shuffle == SHUFFLE_SPACE:
        y = R.spatial_up(x, {"net.0.weight": wb.reshape(wb.shape[0], wb.shape[1], 1, 1), "net.0.bias": b}, "")
    elif shuffle == SHUFFLE_TIME:
        y = R.time_up(x, {"net.0.weight": wb.reshape(wb.shape[0], wb.shape[1], 1), "net.0.bias": b}, "")
    elif stride == (1, 2, 2):
        y = R.spatial_down(x, {"conv.weight": wb, "conv.bias": b}, "")
    elif stride == (2, 1, 1):
        y = R.time_down(x, {"conv.weight": wb, "conv.bias": b}, "")
    else:
        k = tuple(k3) if k3 is not None else (1,) * (5 - wb.ndim) + tuple(wb.shape[2:])
        y = R.causal_conv3d(x, wb.reshape(wb.shape[0], wb.shape[1], *k), b)
        if act == ACT_ELU:
            y = F.elu(y)
        elif act == ACT_SILU:
            y = F.silu(y)
    if res is not None:
        y = y + res.float().cpu().permute(0, 4, 1, 2, 3)
    return y.permute(0, 2, 3, 4, 1).contiguous()


def _check_vs_oracle(name, y, ref):
    """bf16 result vs the fp32 oracle: fp32 accumulation of bf16 products is exact to ~1e-6 relative, so the whole error
    budget is the single rounding of the output to bf16 (half an ulp = 2^-9 relative) plus the MUFU activations."""
    a = y.float().cpu()
    assert a.shape == ref.shape, (a.shape, ref.shape)
    err = (a - ref).abs()
    bound = ref.abs() * 2.0 ** -8 + 2e-3
    worst = (err - bound).max().item()
    assert worst <= 0, f"{name}: |err| exceeds one bf16 ulp of the oracle value by {worst}"
    assert err.mean().item() <= 0.0015 * ref.abs().mean().item() + 1e-4, (name, err.mean().item())


def _engine():
    m = VideoTokenizer(image_size=32, init_dim=16, codebook_size=1024, layers=("residual",)).cuda().bfloat16()
    return m.engine


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tc_matches_cuda_core(case):
    assert torch.cuda.is_available()
    name, wshape, k3, xshape, kw, q = case
    kw = dict(kw)
    g = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    fan_in = 1
    for v in wshape[1:]:
        fan_in *= v
    w = (torch.randn(wshape, generator=g) * fan_in ** -0.5).cuda()
    bias = (torch.randn(wshape[0], generator=g) * 0.1).cuda()
    B, T, H, W = xshape
    x = torch.randn((B, T, H, W, wshape[1]), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    pk = pack_conv(w, bias, torch.bfloat16, k=k3, shuffle_q=q)
    down = kw.pop("down", None)
    if down == "space":
        kw["out_spatial"] = (T, (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1)
    elif down == "time":
        kw["out_spatial"] = ((T + 2 - 3) // 2 + 1, H, W)
    want_res = kw.pop("res", False)

    def run(use_tc):
        eng.use_tc = use_tc
        res = None
        if want_res:
            To, Ho, Wo = kw.get("out_spatial", (T, H, W))
            gg = torch.Generator(device="cpu").manual_seed(7)
            res = torch.randn((B, To, Ho, Wo, wshape[0]), generator=gg).cuda().to(torch.bfloat16)
        return eng.conv(x, pk, res=res, **kw)

    eng.tc_calls = 0
    eng.tc_variant = "tap"
    y_tc = run(True)
    assert eng.tc_calls == 1, "wgmma path was not taken"
    y_ref = run(False)
    torch.cuda.synchronize()
    res_o = None
    if want_res:
        To, Ho, Wo = kw.get("out_spatial", (T, H, W))
        res_o = torch.randn((B, To, Ho, Wo, wshape[0]), generator=torch.Generator(device="cpu").manual_seed(7)).to(torch.bfloat16)
    _check_vs_oracle(name, y_tc, _oracle_conv(w, bias, x, k3, kw, res_o))
    assert y_tc.shape == y_ref.shape
    a, b = y_tc.float(), y_ref.float()
    assert torch.isfinite(a).all()
    tol = 0.008 * b.abs().max().item() + 1e-3          # one bf16 ulp at the output scale
    err = (a - b).abs().max().item()
    assert err <= tol, f"{name}: max-abs diff {err} > {tol}"
    assert (a - b).abs().mean().item() < 0.002 * b.abs().mean().item() + 1e-4


SLAB_CASES = [
    ("slab_c64_32x32", (64, 64, 3, 3, 3), (1, 3, 32, 32), dict(act=ACT_ELU)),
    ("slab_c64_w128", (64, 64, 3, 3, 3), (1, 2, 16, 128), dict(act=ACT_ELU)),
    ("slab_c128_64x64_b2", (128, 128, 3, 3, 3), (2, 3, 64, 64), dict(act=ACT_ELU)),
    ("slab_c256_32x32", (256, 256, 3, 3, 3), (1, 4, 32, 32), dict()),
    ("slab_c512_16x16", (512, 512, 3, 3, 3), (2, 5, 16, 16), dict(act=ACT_ELU)),
    ("slab_c512_16x16_T10", (512, 512, 3, 3, 3), (1, 10, 16, 16), dict(act=ACT_ELU)),
    ("slab_ragged_24x20", (64, 64, 3, 3, 3), (1, 3, 24, 20), dict(act=ACT_ELU)),
    ("slab_small_8x8", (128, 64, 3, 3, 3), (2, 3, 8, 8), dict()),
    ("slab_res", (64, 64, 3, 3, 3), (1, 2, 32, 32), dict(res=True)),
    ("slab_k133", (64, 64, 1, 3, 3), (1, 3, 32, 32), dict()),
    ("slab_pointwise_c64", (64, 64, 1, 1, 1), (2, 3, 32, 32), dict(act=ACT_ELU)),
    ("slab_pointwise_c512_res", (512, 512, 1, 1, 1), (1, 4, 16, 16), dict(res=True)),
    ("slab_linear_512_768", (768, 512, 1, 1, 1), (1, 2, 16, 16), dict()),
    ("slab_conv_out_co3", (3, 64, 3, 3, 3), (1, 3, 16, 32), dict()),
    ("slab_co16", (16, 64, 3, 3, 3), (1, 2, 16, 16), dict(act=ACT_ELU)),
    ("slab_up_space", (256, 128, 1, 1), (1, 3, 16, 16), dict(act=ACT_SILU, shuffle=SHUFFLE_SPACE, q=4)),
    ("slab_up_time", (1024, 512, 1), (1, 3, 8, 8), dict(act=ACT_SILU, shuffle=SHUFFLE_TIME, q=2, k3=(1, 1, 1))),
]


@pytest.mark.parametrize("case", SLAB_CASES, ids=[c[0] for c in SLAB_CASES])
def test_slab_matches_cuda_core(case):
    assert torch.cuda.is_available()
    name, wshape, xshape, kw = case
    kw = dict(kw)
    g = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    fan_in = 1
    for v in wshape[1:]:
        fan_in *= v
    w = (torch.randn(wshape, generator=g) * fan_in ** -0.5).cuda()
    bias = (torch.randn(wshape[0], generator=g) * 0.1).cuda()
    B, T, H, W = xshape
    x = torch.randn((B, T, H, W, wshape[1]), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    k3 = kw.pop("k3", None)
    pk = pack_conv(w, bias, torch.bfloat16, k=k3, shuffle_q=kw.pop("q", 1))
    want_res = kw.pop("res", False)
    res = torch.randn((B, T, H, W, wshape[0]), generator=g).cuda().to(torch.bfloat16) if want_res else None
    eng.use_tc, eng.tc_variant, eng.slab_calls = True, "auto", 0
    y_slab = eng.conv(x, pk, res=res, **kw)
    assert eng.slab_calls == 1, "slab kernel was not taken"
    eng.tc_variant = "tap"
    y_tap = eng.conv(x, pk, res=res, **kw)
    eng.use_tc = False
    y_ref = eng.conv(x, pk, res=res, **kw)
    torch.cuda.synchronize()
    _check_vs_oracle(name, y_slab, _oracle_conv(w, bias, x, k3, kw, res))
    a, b, c = y_slab.float(), y_ref.float(), y_tap.float()
    assert torch.isfinite(a).all()
    tol = 0.008 * b.abs().max().item() + 1e-3
    err = (a - b).abs().max().item()
    assert err <= tol, f"{name}: slab vs cuda-core max-abs diff {err} > {tol}"
    assert (a - c).abs().max().item() <= tol


@pytest.mark.parametrize("C_,tshift", [(256, False), (512, True), (64, False)])
def test_fused_geglu_feed_forward_matches_cuda_core(C_, tshift):
    """fc1 + GEGLU fused in the wgmma epilogue (hidden width padded to 64) + fc2 vs the unfused CUDA-core path."""
    from magvit2_pytorch_b200.engine import pack_ff
    assert torch.cuda.is_available()
    g = torch.Generator(device="cpu").manual_seed(C_)
    I = int(C_ * 4 * 2 / 3)
    w1 = (torch.randn((2 * I, C_, 1, 1, 1), generator=g) * C_ ** -0.5).cuda()
    b1 = (torch.randn(2 * I, generator=g) * 0.1).cuda()
    w2 = (torch.randn((C_, I, 1, 1, 1), generator=g) * I ** -0.5).cuda()
    b2 = (torch.randn(C_, generator=g) * 0.1).cuda()
    fc1, fc2 = pack_ff(w1, b1, w2, b2, torch.bfloat16)
    p = dict(gamma=torch.ones(C_, device="cuda"), fc1=fc1, fc2=fc2, inner=I)
    x = torch.randn((2, 3, 8, 8, C_), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    eng.use_tc, eng.tc_calls = True, 0
    y_tc = eng.feed_forward(x, p, token_shift=tshift)
    assert eng.tc_calls == 2
    eng.use_tc = False
    y_ref = eng.feed_forward(x, p, token_shift=tshift)
    torch.cuda.synchronize()
    a, b = y_tc.float(), y_ref.float()
    assert torch.isfinite(a).all()
    # the unfused path rounds the hidden activations to bf16 twice (fc1 output, GEGLU output); the fused one once
    assert (a - b).abs().max().item() <= 0.02 * b.abs().max().item() + 2e-3
    assert (a - b).abs().mean().item() <= 0.004 * b.abs().mean().item() + 1e-4


@pytest.mark.parametrize("variant", ["tap", "auto"])
def test_conv_in_kwpack_matches_cuda_core(variant):
    """conv_in (7x7x7, C_in=3) through mv2_ingest_kwpack + wgmma (49 taps x 32 packed channels) vs the CUDA-core conv."""
    assert torch.cuda.is_available()
    m = VideoTokenizer(image_size=32, init_dim=64, codebook_size=1024, layers=("residual",)).cuda().bfloat16()
    eng = m.engine
    g = torch.Generator(device="cpu").manual_seed(3)
    v = torch.randn((2, 3, 5, 32, 32), generator=g).cuda()
    pin = eng._packs["conv_in_tc"]
    assert pin is not None
    eng.use_tc, eng.tc_calls, eng.slab_calls, eng.tc_variant = True, 0, 0, variant
    x = eng.ingest_kwpack(v, 2, pin)
    y_tc = eng.conv(x, pin, pad=(6, 3, 0))
    assert eng.tc_calls == 1 and eng.slab_calls == (1 if variant == "auto" else 0)
    eng.use_tc = False
    y_ref = eng.conv(eng.to_channels_last(v, 2), eng._packs["conv_in"])
    torch.cuda.synchronize()
    a, b = y_tc.float(), y_ref.float()
    assert a.shape == b.shape
    assert (a - b).abs().max().item() <= 0.008 * b.abs().max().item() + 1e-3


@pytest.mark.parametrize("L,D,heads,nseq", [(256, 32, 8, 6), (100, 32, 4, 3), (1024, 32, 2, 2), (128, 64, 4, 2),
                                            (64, 32, 4, 2), (65, 64, 2, 3), (129, 32, 3, 2)])
def test_attention_tensor_core_kernel_matches_fp32_cuda_core(L, D, heads, nseq):
    """bf16 mma.sync flash-attention kernel (space attention) vs the fp32 CUDA-core attention kernel on the same
    (bf16-representable) inputs; L = 64 is the smallest sequence it takes, 65 and 129 leave a partial 128-query block."""
    import ctypes as C
    from magvit2_pytorch_b200 import _lib
    from magvit2_pytorch_b200._lib import AttnArgs, check
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(L + D)
    HD = heads * D
    qkv = (torch.randn((nseq * L, 3 * HD), generator=g) * 1.5).to(torch.bfloat16).cuda()
    mem = torch.randn((2, heads, 4, D), generator=g).to(torch.bfloat16).float().cuda()
    outs = {}
    for dt, code in ((torch.bfloat16, 1), (torch.float32, 0)):
        x = qkv.to(dt).contiguous()
        o = torch.empty((nseq * L, HD), device="cuda", dtype=dt)
        a = AttnArgs(qkv=x.data_ptr(), out=o.data_ptr(), mem_kv=mem.data_ptr(), dtype=code, heads=heads, dim_head=D,
                     n_mem=4, causal=0, n_outer=nseq, n_inner=1, L=L, outer_stride=L, inner_stride=0, tok_stride=1)
        check(lib.mv2_attention(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "mv2_attention")
        outs[dt] = o.float()
    torch.cuda.synchronize()
    a_, b_ = outs[torch.bfloat16], outs[torch.float32]
    assert torch.isfinite(a_).all()
    assert (a_ - b_).abs().max().item() < 0.03 * b_.abs().max().item() + 5e-3
    assert (a_ - b_).abs().mean().item() < 0.006 * b_.abs().mean().item() + 1e-3
    # the CPU oracle's Attend restatement (A:218-241 with the 4 memory key/values prepended, M:383-385) on the same inputs
    t = qkv.float().cpu().reshape(nseq, L, 3, heads, D).permute(2, 0, 3, 1, 4)
    memc = mem.cpu()
    k_ = torch.cat((memc[0][None].expand(nseq, -1, -1, -1), t[1]), dim=-2)
    v_ = torch.cat((memc[1][None].expand(nseq, -1, -1, -1), t[2]), dim=-2)
    o_ = R.softmax_attention(t[0], k_, v_, causal=False).permute(0, 2, 1, 3).reshape(nseq * L, HD)
    assert (b_.cpu() - o_).abs().max().item() < 2e-5 * o_.abs().max().item() + 2e-5          # fp32 kernel vs oracle
    assert (a_.cpu() - o_).abs().max().item() < 0.03 * o_.abs().max().item() + 5e-3          # bf16 mma kernel vs oracle
    assert (a_.cpu() - o_).abs().mean().item() < 0.006 * o_.abs().mean().item() + 1e-3


@pytest.mark.parametrize("L,heads,nseq", [(1024, 16, 3), (200, 4, 2), (4096, 2, 1), (1, 4, 3), (257, 8, 2)])
def test_linear_attention_tensor_core_kernels_match_fp32_cuda_core(L, heads, nseq):
    """bf16 mma.sync Taylor-linear-attention kernels vs the fp32 CUDA-core kernels on the same bf16-representable inputs."""
    import ctypes as C
    from magvit2_pytorch_b200 import _lib
    from magvit2_pytorch_b200._lib import check
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(L + heads)
    HD = heads * 8
    q = (torch.randn((nseq * L, HD), generator=g)).to(torch.bfloat16).cuda()
    kv = (torch.randn((nseq * L, 2 * HD), generator=g)).to(torch.bfloat16).cuda()
    outs = {}
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for dt, code in ((torch.bfloat16, 1), (torch.float32, 0)):
        ws = torch.empty(lib.mv2_linattn_workspace_bytes(nseq, heads, L) // 4, device="cuda", dtype=torch.float32)
        qq, kk = q.to(dt).contiguous(), kv.to(dt).contiguous()
        o = torch.empty((nseq * L, HD), device="cuda", dtype=dt)
        check(lib.mv2_linear_attention(qq.data_ptr(), kk.data_ptr(), o.data_ptr(), code, nseq, L, heads, 8, ws.data_ptr(), st),
              "mv2_linear_attention")
        outs[dt] = o.float()
    torch.cuda.synchronize()
    a_, b_ = outs[torch.bfloat16], outs[torch.float32]
    assert torch.isfinite(a_).all()
    assert (a_ - b_).abs().max().item() < 0.04 * b_.abs().max().item() + 5e-3
    assert (a_ - b_).abs().mean().item() < 0.01 * b_.abs().mean().item() + 1e-3
    # the CPU oracle's Taylor-attention restatement (Appendix A.3) with identity projections = the bare core
    eye = torch.eye(HD)
    sd = {"attn.to_q.0.weight": torch.cat((eye, torch.zeros(HD, 2 * HD)), dim=1),
          "attn.to_kv.0.weight": torch.cat((torch.zeros(2 * HD, HD), torch.eye(2 * HD)), dim=1),
          "attn.to_out.0.weight": eye}
    xin = torch.cat((q.float().cpu(), kv.float().cpu()), dim=-1).reshape(nseq, L, 3 * HD)
    o_ = R.taylor_linear_attention(xin, sd, "", heads, 8).reshape(nseq * L, HD)
    assert (b_.cpu() - o_).abs().max().item() < 1e-4 * o_.abs().max().item() + 1e-4
    assert (a_.cpu() - o_).abs().max().item() < 0.04 * o_.abs().max().item() + 5e-3
    assert (a_.cpu() - o_).abs().mean().item() < 0.01 * o_.abs().mean().item() + 1e-3


RU_CASES = [
    # name, C, (B, T, H, W)
    ("ru_c64_mw4_small", 64, (1, 3, 32, 32)),
    ("ru_c64_mw2_w16", 64, (2, 3, 16, 16)),
    ("ru_c128_small", 128, (1, 4, 16, 32)),
    ("ru_c64_ragged_24x20", 64, (1, 3, 24, 20)),
    ("ru_c128_ragged_20x24", 128, (2, 3, 20, 24)),
    ("ru_c64_multi_tile_per_cta", 64, (1, 10, 128, 128)),      # 320 tiles: 2-3 tiles per persistent CTA
    ("ru_c128_multi_tile_per_cta", 128, (2, 5, 64, 64)),       # 320 tiles
]


def _ru_pack(C_, g):
    w3 = (torch.randn((C_, C_, 3, 3, 3), generator=g) * (27 * C_) ** -0.5).cuda()
    b3 = (torch.randn(C_, generator=g) * 0.1).cuda()
    w1 = (torch.randn((C_, C_, 1, 1, 1), generator=g) * C_ ** -0.5).cuda()
    b1 = (torch.randn(C_, generator=g) * 0.1).cuda()
    hd = max(16, C_ // 2)
    wk = (torch.randn(C_, generator=g) * C_ ** -0.5).cuda()
    bk = float(torch.randn(1, generator=g).item() * 0.1)
    sw1 = (torch.randn((hd, C_), generator=g) * C_ ** -0.5).cuda()
    sb1 = (torch.randn(hd, generator=g) * 0.1).cuda()
    sw2 = (torch.randn((C_, hd), generator=g) * hd ** -0.5).cuda()
    sb2 = (torch.randn(C_, generator=g) * 0.1).cuda()
    p = dict(conv3=pack_conv(w3, b3, torch.bfloat16), conv1=pack_conv(w1, b1, torch.bfloat16), wk=wk.contiguous(), bk=bk,
             w1=sw1.contiguous(), b1=sb1, w2=sw2.contiguous(), b2=sb2, hidden=hd)
    sd = {"fn.0.conv.weight": w3.to(torch.bfloat16).float().cpu(), "fn.0.conv.bias": b3.cpu(),
          "fn.2.weight": w1.to(torch.bfloat16).float().cpu(), "fn.2.bias": b1.cpu(),
          "fn.4.to_k.weight": wk.cpu().reshape(1, C_, 1, 1), "fn.4.to_k.bias": torch.tensor([bk]),
          "fn.4.net.0.weight": sw1.cpu().reshape(hd, C_, 1, 1), "fn.4.net.0.bias": sb1.cpu(),
          "fn.4.net.2.weight": sw2.cpu().reshape(C_, hd, 1, 1), "fn.4.net.2.bias": sb2.cpu()}
    return p, sd


@pytest.mark.parametrize("case", RU_CASES, ids=[c[0] for c in RU_CASES])
def test_fused_residual_unit(case):
    """mv2_tc_ru_forward (conv3x3x3 + ELU + conv1x1x1 + ELU + SE pool records in one wgmma launch) + gate + residual
    against (a) the unfused kernels on identical inputs and (b) the CPU oracle's residual_unit (M:930-944)."""
    assert torch.cuda.is_available()
    name, C_, (B, T, H, W) = case
    g = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    p, sd = _ru_pack(C_, g)
    x = torch.randn((B, T, H, W, C_), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    eng.use_tc, eng.tc_variant = True, "auto"
    eng.fuse_ru, eng.fused_ru_calls = True, 0
    out_f = eng.residual_unit(x, p)
    assert eng.fused_ru_calls == 1, "fused kernel was not taken"
    eng.fuse_ru = False
    out_u = eng.residual_unit(x, p)
    torch.cuda.synchronize()
    eng.fuse_ru = True
    a, b = out_f.float().cpu(), out_u.float().cpu()
    assert torch.isfinite(a).all()
    # same bf16 operands and fp32 accumulation in both paths; only the SE pooling order differs (fp32 round-off in the gate)
    assert (a - b).abs().max().item() <= 2.0 ** -7 * b.abs().max().item() + 1e-3, (name, (a - b).abs().max().item())
    assert (a != b).float().mean().item() < 0.02, (name, (a != b).float().mean().item())
    ref = R.residual_unit(x.float().cpu().permute(0, 4, 1, 2, 3).contiguous(), sd, "").permute(0, 2, 3, 4, 1)
    err = (a - ref).abs()
    # three bf16 roundings along the unit (h, y, out) against the fp32 oracle
    assert err.max().item() <= 0.02 * ref.abs().max().item() + 5e-3, (name, err.max().item())
    assert err.mean().item() <= 0.004 * ref.abs().mean().item() + 2e-4, (name, err.mean().item())


@pytest.mark.parametrize("T,tp,H,W", [(6, 3, 32, 32), (5, 1, 16, 24), (4, 0, 16, 16)])
def test_conv_out_channels_first_with_cropped_frames(T, tp, H, W):
    """conv_out (Co = 3) writing torch's (B,C,T,H,W) layout directly, without the leading time_padding frames the
    reference drops after the conv (M:1642-1647), vs conv + mv2_to_channels_first crop and vs the CPU oracle."""
    assert torch.cuda.is_available()
    g = torch.Generator(device="cpu").manual_seed(T * 100 + tp)
    w = (torch.randn((3, 64, 3, 3, 3), generator=g) * (27 * 64) ** -0.5).cuda()
    bias = (torch.randn(3, generator=g) * 0.1).cuda()
    x = torch.randn((2, T, H, W, 64), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    pk = pack_conv(w, bias, torch.bfloat16)
    eng.use_tc, eng.tc_variant, eng.slab_calls = True, "auto", 0
    y_cf = eng.conv(x, pk, pad=(2 - tp, 1, 1), out_spatial=(T - tp, H, W), out_cf=True)
    assert eng.slab_calls == 1 and y_cf.shape == (2, 3, T - tp, H, W)
    y_ref = eng.to_channels_first(eng.conv(x, pk), t_crop=tp)
    torch.cuda.synchronize()
    assert torch.equal(y_cf, y_ref)
    ref = _oracle_conv(w, bias, x, None, {}).permute(0, 4, 1, 2, 3)[:, :, tp:]
    _check_vs_oracle("conv_out_cf", y_cf.permute(0, 2, 3, 4, 1), ref.permute(0, 2, 3, 4, 1).contiguous())


@pytest.mark.parametrize("C_,shape", [(512, (2, 3, 16, 16)), (256, (1, 4, 8, 8)), (64, (2, 2, 5, 7)), (1024, (1, 2, 8, 8)), (24, (1, 3, 6, 6))])
def test_unfused_residual_unit_vs_oracle(C_, shape):
    """The unfused ResidualUnit path (conv3x3x3 + ELU and conv1x1x1 + ELU on the tensor cores, then SE pool, gate MLP and
    gate/residual as separate launches; C = 24 takes the generic bf16 se_pool kernel) against the CPU oracle's
    residual_unit (M:930-944, M:221-240)."""
    assert torch.cuda.is_available()
    B, T, H, W = shape
    g = torch.Generator(device="cpu").manual_seed(C_ + H)
    p, sd = _ru_pack(C_, g)
    for k in ("w1", "w2"):                       # a bf16 model's SE weights are bf16 values
        p[k] = p[k].to(torch.bfloat16).float().contiguous()
    sd["fn.4.net.0.weight"] = p["w1"].cpu().reshape(-1, C_, 1, 1)
    sd["fn.4.net.2.weight"] = p["w2"].cpu().reshape(C_, -1, 1, 1)
    x = torch.randn((B, T, H, W, C_), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    eng.use_tc, eng.tc_variant, eng.fuse_ru, eng.fused_ru_calls = True, "auto", False, 0
    out = eng.residual_unit(x, p)
    torch.cuda.synchronize()
    assert eng.fused_ru_calls == 0
    a = out.float().cpu()
    assert torch.isfinite(a).all()
    ref = R.residual_unit(x.float().cpu().permute(0, 4, 1, 2, 3).contiguous(), sd, "").permute(0, 2, 3, 4, 1)
    err = (a - ref).abs()
    assert err.max().item() <= 0.02 * ref.abs().max().item() + 5e-3, err.max().item()
    assert err.mean().item() <= 0.004 * ref.abs().mean().item() + 2e-4, err.mean().item()


@pytest.mark.parametrize("C_,Co,shape", [(512, 512, (2, 10, 16, 16)), (64, 128, (1, 5, 8, 16)), (128, 128, (2, 4, 16, 24)), (512, 512, (4, 20, 16, 16))])
def test_slab_time_downsample(C_, Co, shape):
    """TimeDownsample2x (F.pad(2,0) + Conv1d k3 s2 along t, M:796-807) on the slab kernel (t-strided slab loads) vs the
    tap-wise kernel, the CUDA-core kernel and the CPU oracle."""
    assert torch.cuda.is_available()
    B, T, H, W = shape
    g = torch.Generator(device="cpu").manual_seed(C_ + T)
    w = (torch.randn((Co, C_, 3), generator=g) * (3 * C_) ** -0.5).cuda()
    bias = (torch.randn(Co, generator=g) * 0.1).cuda()
    x = torch.randn((B, T, H, W, C_), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    pk = pack_conv(w, bias, torch.bfloat16, k=(3, 1, 1))
    kw = dict(stride=(2, 1, 1), pad=(2, 0, 0), out_spatial=((T + 2 - 3) // 2 + 1, H, W))
    eng.use_tc, eng.tc_variant, eng.slab_calls = True, "auto", 0
    y_slab = eng.conv(x, pk, **kw)
    assert eng.slab_calls == 1, "slab kernel was not taken"
    eng.tc_variant = "tap"
    y_tap = eng.conv(x, pk, **kw)
    torch.cuda.synchronize()
    eng.tc_variant = "auto"
    _check_vs_oracle("slab_down_time", y_slab, _oracle_conv(w, bias, x, (3, 1, 1), dict(stride=(2, 1, 1))))
    assert (y_slab.float() - y_tap.float()).abs().max().item() <= 0.008 * y_tap.float().abs().max().item() + 1e-3


@pytest.mark.parametrize("Ci,Co,shape", [(64, 128, (2, 3, 32, 32)), (128, 256, (1, 4, 64, 64)), (256, 512, (2, 3, 32, 32)),
                                         (64, 128, (1, 2, 24, 40)), (64, 64, (1, 2, 16, 64)), (64, 128, (4, 20, 128, 128))])
def test_slab_space_downsample(Ci, Co, shape):
    """SpatialDownsample2x (Conv2d k3 s2 p1 per frame, M:770-780) on the slab kernel (row-parity sub-slabs of the (W/2) x (2C)
    view, mv2_tc_down_space_forward) vs the tap-wise kernel and the CPU oracle."""
    from magvit2_pytorch_b200.engine import pack_conv_down_space
    assert torch.cuda.is_available()
    B, T, H, W = shape
    g = torch.Generator(device="cpu").manual_seed(Ci + Co + H)
    w = (torch.randn((Co, Ci, 3, 3), generator=g) * (9 * Ci) ** -0.5).cuda()
    bias = (torch.randn(Co, generator=g) * 0.1).cuda()
    x = torch.randn((B, T, H, W, Ci), generator=g).cuda().to(torch.bfloat16)
    eng = _engine()
    pk = pack_conv(w, bias, torch.bfloat16)
    pack_conv_down_space(pk, w)
    assert pk.w_down is not None
    kw = dict(stride=(1, 2, 2), pad=(0, 1, 1), out_spatial=(T, H // 2, W // 2))
    eng.use_tc, eng.tc_variant, eng.slab_calls = True, "auto", 0
    y_slab = eng.conv(x, pk, **kw)
    assert eng.slab_calls == 1, "slab down-space kernel was not taken"
    eng.tc_variant = "tap"
    y_tap = eng.conv(x, pk, **kw)
    torch.cuda.synchronize()
    eng.tc_variant = "auto"
    assert (y_slab.float() - y_tap.float()).abs().max().item() <= 0.008 * y_tap.float().abs().max().item() + 1e-3
    if B * T * H * W <= 65536:       # the CPU oracle on the small cases
        _check_vs_oracle("slab_down_space", y_slab, _oracle_conv(w, bias, x, None, dict(stride=(1, 2, 2))))


@pytest.mark.parametrize("T,HW,D,heads,causal,n_mem", [
    pytest.param(5, 64, 32, 8, 1, 4, id="5-64-32-8-1"), pytest.param(1, 16, 32, 4, 1, 4, id="1-16-32-4-1"),
    pytest.param(8, 24, 64, 2, 1, 4, id="8-24-64-2-1"), pytest.param(3, 10, 32, 3, 0, 4, id="3-10-32-3-0"),
    # more than 8 frames or memory slots, or dim_head 96: the general kernel (attention_kernel<bf16, D / 32>)
    pytest.param(9, 16, 32, 4, 1, 0, id="9-16-32-4-1-nmem0"), pytest.param(33, 8, 64, 2, 1, 9, id="33-8-64-2-1-nmem9"),
    pytest.param(5, 12, 96, 2, 1, 4, id="5-12-96-2-1"), pytest.param(9, 6, 96, 3, 1, 9, id="9-6-96-3-1-nmem9"),
])
def test_attention_small_sequences_kernel(T, HW, D, heads, causal, n_mem):
    """Short-sequence attention kernel (time attention: one warp per (pixel, head), right-aligned causal mask over n_mem
    memory key/values + the frames so far, A:46-47 / A:123-129; masking off when L == 1, A:209-210) vs the fp32 general
    kernel and the CPU oracle, with the strided token addressing of TimeAttention (M:456-464).  Sequences the short kernel
    cannot hold take the general kernel in bf16 as well."""
    import ctypes as C
    from magvit2_pytorch_b200 import _lib
    from magvit2_pytorch_b200._lib import AttnArgs, check
    lib = _lib.load()
    B = 2
    g = torch.Generator(device="cpu").manual_seed(T * 10 + D)
    HDm = heads * D
    qkv = (torch.randn((B * T * HW, 3 * HDm), generator=g) * 1.2).to(torch.bfloat16).cuda()
    mem = torch.randn((2, heads, n_mem, D), generator=g).to(torch.bfloat16).float().cuda()
    mem_buf = mem if n_mem > 0 else torch.zeros(1, device="cuda")       # the library takes a non-null mem_kv pointer
    outs = {}
    for dt, code in ((torch.bfloat16, 1), (torch.float32, 0)):
        x = qkv.to(dt).contiguous()
        o = torch.zeros((B * T * HW, HDm), device="cuda", dtype=dt)
        a = AttnArgs(qkv=x.data_ptr(), out=o.data_ptr(), mem_kv=mem_buf.data_ptr(), dtype=code, heads=heads, dim_head=D,
                     n_mem=n_mem, causal=causal, n_outer=B, n_inner=HW, L=T, outer_stride=T * HW, inner_stride=1,
                     tok_stride=HW)
        check(lib.mv2_attention(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "mv2_attention")
        outs[dt] = o.float().cpu()
    torch.cuda.synchronize()
    t = qkv.float().cpu().reshape(B, T, HW, 3, heads, D).permute(3, 0, 2, 4, 1, 5).reshape(3, B * HW, heads, T, D)
    memc = mem.cpu()
    k_ = torch.cat((memc[0][None].expand(B * HW, -1, -1, -1), t[1]), dim=-2)
    v_ = torch.cat((memc[1][None].expand(B * HW, -1, -1, -1), t[2]), dim=-2)
    o_ = R.softmax_attention(t[0], k_, v_, causal=bool(causal))                    # (B*HW, heads, T, D)
    o_ = o_.reshape(B, HW, heads, T, D).permute(0, 3, 1, 2, 4).reshape(B * T * HW, HDm)
    a_, b_ = outs[torch.bfloat16], outs[torch.float32]
    assert (b_ - o_).abs().max().item() < 2e-5 * o_.abs().max().item() + 2e-5
    assert (a_ - o_).abs().max().item() < 2.0 ** -8 * o_.abs().max().item() + 2e-3     # one bf16 rounding of the output


# (kt, stride, cin, cout, then): `then` is done after a first forward and before the checked one -- "new_bias": a bias
# assigned through .data (new storage, same version counter); "copy": the module deep-copied and pickled
CONV_T_CASES = [(3, 2, 64, 64, None), (4, 2, 64, 32, None), (3, 1, 64, 64, None), (3, 2, 5, 4, None),
                (3, 2, 64, 64, "new_bias"), (3, 2, 64, 64, "copy")]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kt,stride,cin,cout,then",
                         [pytest.param(*c, id="-".join(str(v) for v in c if v is not None)) for c in CONV_T_CASES])
def test_causal_conv_transpose3d_vs_oracle(dtype, kt, stride, cin, cout, then):
    """CausalConvTranspose3d (M:990-1024) on the device (one causal conv + depth-to-time) against the CPU restatement."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import copy
    import pickle
    from magvit2_pytorch_b200.modules import CausalConvTranspose3d
    from oracle.restated import causal_conv_transpose3d
    torch.manual_seed(kt + stride + cin)
    m = CausalConvTranspose3d(cin, cout, (kt, 3, 3), time_stride=stride)
    x = torch.randn(2, cin, 5, 16, 16)
    bias = torch.randn(cout)
    if dtype == torch.bfloat16:                # identical bf16-representable operands on both sides
        with torch.no_grad():
            m.conv.weight.copy_(m.conv.weight.bfloat16().float()); m.conv.bias.copy_(m.conv.bias.bfloat16().float())
        x, bias = x.bfloat16().float(), bias.bfloat16().float()
    m = m.cuda().to(dtype)
    xd = x.cuda().to(dtype)
    mods = [m]
    if then is not None:
        m(xd)                                  # packs
    if then == "new_bias":
        m.conv.bias.data = bias.cuda().to(dtype)
    elif then == "copy":
        mods = [copy.deepcopy(m), pickle.loads(pickle.dumps(m))]
    want = causal_conv_transpose3d(x, m.conv.weight.detach().float().cpu(), m.conv.bias.detach().float().cpu(), stride)
    outs = [mod(xd).float().cpu() for mod in mods]
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    for got in outs:
        assert got.shape == want.shape
        assert (got - want).abs().max().item() < tol * max(1.0, want.abs().max().item())
        assert torch.equal(got, outs[0])
