"""Attention dropout on the device: mv2_attention_dropout_mask against the numpy replica (tests/attn_dropout_ref.py) bit for bit,
mv2_attention_dropout against a float64 softmax that applies the replica's mask, the mask's statistics, and the tokenizer:
eval outputs untouched by attn_dropout, training gradients against the float64 oracle with the same masks, and
reproducibility from torch's seed.

Forward bound.  o = s sum_j keep_j w_j v_j with s = fp32(1 / (1 - p)) and the undropped softmax weights w (the denominator
is undropped).  The kernels' rounding is that of mv2_attention (tests/test_attention_gpu.py, _softmax64) with the numerator
sums restricted to the kept keys: the relative error eps_j of each p_j enters the numerator as s sum_j keep_j w_j eps_j |v_j|
and the denominator as sum_j w_j eps_j |o|; the sums gamma_c(M + n_t + 5) (s sum_j keep_j w_j |v_j| + |o|); the mma kernel's
bf16 P in the numerator 2^-8 s sum_j keep_j w_j |v_j|; the final s / l, its product and one more rounding for s: 3u |o|."""
import ctypes as C
import math
import re
import zlib

import numpy as np
import pytest
import torch

from tests.attn_dropout_ref import dropout_scale, keep_mask
from tests.test_attention_gpu import (ATTN_CASES, DEV, DT, KPROP, R_EXP, U_BF16, _attn_id, _attn_setup, _kind, _short,
                                      _softmax64, guard)  # noqa: F401  (guard: the fixture)
from tests.test_conv_grad_gpu import _gamma
from tests.test_simt_ops_gpu import U, _check, _rejects
from tests.util import build_oracle, build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu
E_ARG = -1


def _lib():
    from magvit2_pytorch_b200 import _lib as L
    return L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dargs(seed, call, p):
    from magvit2_pytorch_b200._lib import DropoutArgs
    return DropoutArgs(seed=seed, call=call, p=p)


def _device_mask(n_seq, heads, L, n_mem, seed, call, p):
    from magvit2_pytorch_b200._lib import check
    keep = torch.full((n_seq, heads, L, n_mem + L), 7, dtype=torch.uint8, device=DEV)
    check(_lib().mv2_attention_dropout_mask(n_seq, heads, L, n_mem, C.byref(_dargs(seed, call, p)), keep.data_ptr(), _st()),
          "mv2_attention_dropout_mask")
    return keep


def _twin(kernel):
    return kernel.replace("_kernel<", "_dropout_kernel<")


# ------------------------------------------------------------------------------------------------------------------
# the mask
# ------------------------------------------------------------------------------------------------------------------
# (n_seq, heads, L, n_mem): the space layout (n_seq = B T, L = H W) and the time layout (n_seq = B H W, L = T, causal: the mask
# has no causal argument, the entries a causal mask hides are written and compared too), and n_seq past 65536
MASK_SHAPES = [(6, 8, 256, m) for m in (0, 4, 9, 33)] + [(300, 8, 5, m) for m in (0, 4, 9, 33)] + [(70001, 1, 3, 4), (65537, 2, 1, 0)]
MASK_KEYS = [(0, 0, 0.1), (0x0123456789ABCDEF, 1, 0.5), (2 ** 64 - 1, 65535, 0.3), (0xFFFFFFFF00000000, 7, 1 - 2.0 ** -24),
             (12345, 2, 2.0 ** -20)]


@pytest.mark.parametrize("shape", MASK_SHAPES, ids=[f"s{s}-h{h}-L{L}-m{m}" for s, h, L, m in MASK_SHAPES])
def test_mask_kernel_equals_replica(shape):
    for seed, call, p in MASK_KEYS:
        got = _device_mask(*shape, seed, call, p).cpu().numpy()
        want = keep_mask(seed, call, p, *shape)
        assert np.array_equal(got, want), (shape, seed, call, p, int((got != want).sum()))


def test_dropout_argument_checks():
    """Both entry points refuse p outside (0, 1), heads >= 2^16 and call >= 2^16 before launching anything."""
    from magvit2_pytorch_b200._lib import AttnArgs
    lib = _lib()
    buf = torch.full((4,), float("nan"), device=DEV)
    keep = torch.full((4,), 9, dtype=torch.uint8, device=DEV)
    p = buf.data_ptr()
    args = AttnArgs(qkv=p, out=p, mem_kv=p, dtype=1, heads=2, dim_head=32, n_mem=4, causal=0, n_outer=1, n_inner=1, L=64,
                    outer_stride=64, inner_stride=0, tok_stride=1)
    for d in (_dargs(1, 0, 0.), _dargs(1, 0, 1.), _dargs(1, 0, -0.1), _dargs(1, 0, float("nan")), _dargs(1, 65536, 0.1)):
        assert lib.mv2_attention_dropout(C.byref(args), C.byref(d), _st()) == E_ARG
        assert lib.mv2_attention_dropout_mask(1, 2, 1, 0, C.byref(d), keep.data_ptr(), _st()) == E_ARG
    args.heads = 65536
    assert lib.mv2_attention_dropout(C.byref(args), C.byref(_dargs(1, 0, 0.1)), _st()) == E_ARG
    assert lib.mv2_attention_dropout_mask(1, 65536, 1, 0, C.byref(_dargs(1, 0, 0.1)), keep.data_ptr(), _st()) == E_ARG
    assert lib.mv2_attention_dropout(None, C.byref(_dargs(1, 0, 0.1)), _st()) == E_ARG
    assert lib.mv2_attention_dropout(C.byref(args), None, _st()) == E_ARG
    torch.cuda.synchronize()
    assert torch.isnan(buf).all() and (keep == 9).all()


# ------------------------------------------------------------------------------------------------------------------
# the forward against float64
# ------------------------------------------------------------------------------------------------------------------
def _drop64(q, k, v, causal, n_mem, keeps, scale, kernel):
    """float64 dropout attention for each mask of `keeps` ((S,H,L,M) float64); the bound of `kernel` for keeps[0]; and, per
    mask, the largest softmax weight mass (over queries) on which it differs from keeps[0]."""
    S, H, L, D = q.shape
    M = k.shape[2]
    outs = [torch.empty_like(q) for _ in keeps]
    acc = torch.empty_like(q)
    diff = [0.0] * len(keeps)
    i_all = torch.arange(L, device=q.device)[:, None]
    j = torch.arange(M, device=q.device)[None, :]
    masked = causal and L > 1
    lq = max(1, min(L, (1 << 22) // (H * M)))
    kp = KPROP[_kind(kernel)]
    c, n_t = kp["c"], -(-M // kp["tile"])
    e_s = _gamma(D, c) + R_EXP + 4 * U
    g_sum = _gamma(M + n_t + 5, c)
    for s in range(S):
        for q0 in range(0, L, lq):
            i = i_all[q0:q0 + lq]
            valid = (j <= i + n_mem) if masked else torch.ones((i.shape[0], M), dtype=torch.bool, device=q.device)
            qs = q[s, :, q0:q0 + lq]
            sc = (torch.einsum("hid,hjd->hij", qs, k[s]) * D ** -0.5).masked_fill(~valid, -math.inf)
            w = sc.softmax(dim=-1)
            k0 = keeps[0][s, :, q0:q0 + lq]
            for n, kn in enumerate(keeps):
                kn = kn[s, :, q0:q0 + lq]
                outs[n][s, :, q0:q0 + lq] = torch.einsum("hij,hjd->hid", w * kn * scale, v[s])
                diff[n] = max(diff[n], (w * (kn - k0).abs()).sum(-1).max().item())
            A = torch.einsum("hid,hjd->hij", qs.abs(), k[s].abs()) * D ** -0.5
            x = (sc.amax(-1, keepdim=True) - sc).masked_fill(~valid, 0.0)
            e_exp = (3 + 1.173 * x) * 2.0 ** -23 if kp["exp"] == "__expf" else R_EXP
            eps = torch.expm1(e_s * A + U * x + e_exp).masked_fill(~valid, 0.0)
            av, ao = v[s].abs(), outs[0][s, :, q0:q0 + lq].abs()
            we = w * eps
            swk = scale * torch.einsum("hij,hjd->hid", w * k0, av)
            t = scale * torch.einsum("hij,hjd->hid", we * k0, av) + we.sum(-1, keepdim=True) * ao
            t = t + g_sum * (swk + ao) + 3 * U * ao + M * 2.0 ** -125 * (scale * av.amax(-2, keepdim=True) + ao)
            if kp["pround"]:
                t = t + U_BF16 * swk
            acc[s, :, q0:q0 + lq] = (1 + 2.0 ** -6) * t
    return outs, acc, diff


def _run_dropout(call, seed, c, p):
    from magvit2_pytorch_b200._lib import AttnArgs, check
    check(_lib().mv2_attention_dropout(C.byref(AttnArgs(**call.args)), C.byref(_dargs(seed, c, p)), _st()), "mv2_attention_dropout")


DROP_CASES = [(c, p) for c in ATTN_CASES for p in (0.1, 0.5)]


@pytest.mark.parametrize("case,p", DROP_CASES, ids=[f"{_attn_id(c)}-p{p}" for c, p in DROP_CASES])
def test_attention_dropout(case, p, guard):
    """Every mv2_attention case with dropout, against float64 with the replica's mask; the bound rejects the mask shifted by one
    key, with the words j & 3 permuted, and with the memory slots undropped, wherever that moves >= 5% of a query's weight."""
    call = _attn_setup(case, guard)
    seed, ci = 0x9E3779B97F4A7C15 ^ zlib.crc32(_attn_id(case).encode()), 17
    _run_dropout(call, seed, ci, p)
    out = call.result()
    q, k, v = call.operands()
    S, H, L, m = q.shape[0], call.heads, call.lay["L"], call.n_mem
    keep = torch.from_numpy(keep_mask(seed, ci, p, S, H, L, m)).to(DEV).double()
    M = L + m
    perm = torch.arange(M, device=DEV) ^ 1
    perm = torch.where(perm < M, perm, torch.arange(M, device=DEV))
    wrong = {"shifted by one key": keep.roll(1, dims=-1), "words j & 3 permuted": keep[..., perm]}
    if m:
        undrop = keep.clone()
        undrop[..., :m] = 1
        wrong["memory slots undropped"] = undrop
    outs, acc, diff = _drop64(q, k, v, call.causal, m, [keep] + list(wrong.values()), dropout_scale(p), call.kernel)
    dt = DT[call.code]
    _check(out, outs[0], dt, acc, _twin(call.kernel))
    for (what, _), o_w, d in zip(wrong.items(), outs[1:], diff[1:]):
        if d >= 0.05:
            _rejects(out, o_w, dt, acc, f"{_twin(call.kernel)}: mask {what}")


def test_dispatch_under_profiler(guard):
    """Each mv2_attention_dropout call launches the dropout twin of the instance mv2_attention launches for its arguments."""
    from torch.profiler import ProfilerActivity, profile
    calls = [_attn_setup(c, guard) for c in ATTN_CASES]
    want = [_twin(cl.kernel).replace(" ", "") for cl in calls]
    torch.cuda.synchronize()
    # a profiler session that is not the process's first can miss kernels at its start: the calls run twice and the
    # second pass, the last len(want) kernels, is checked
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            for n, cl in enumerate(calls):
                _run_dropout(cl, n, 0, 0.1)
            torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    got = [_short(e.name) for e in evs if re.search(r"attention", e.name)]
    assert len(got) >= len(want) and got[-len(want):] == want, (len(got), len(want))
    assert {g.split("<")[0] for g in got} == {"attention_dropout_kernel", "attention_small_dropout_kernel", "attention_mma_dropout_kernel"}


# ------------------------------------------------------------------------------------------------------------------
# statistics
# ------------------------------------------------------------------------------------------------------------------
def test_mask_statistics():
    """Kept fraction overall, per head and per word j & 3 within 6 sigma of 1 - p; masks of different (seed, call) pairs agree
    at the rate p^2 + (1 - p)^2 within 6 sigma."""
    p, shape = 0.1, (64, 8, 256, 260 - 256)
    keep = _device_mask(*shape, 42, 3, p).double()
    n = keep.numel()

    def near(frac, count, prob, what):
        sig = math.sqrt(prob * (1 - prob) / count)
        assert abs(frac - prob) <= 6 * sig, (what, frac, prob, sig)

    near(keep.mean().item(), n, 1 - p, "overall")
    for h in range(shape[1]):
        near(keep[:, h].mean().item(), n // shape[1], 1 - p, f"head {h}")
    for w in range(4):
        near(keep[..., w::4].mean().item(), keep[..., w::4].numel(), 1 - p, f"word {w}")
    r = p * p + (1 - p) * (1 - p)
    for seed, call in ((42, 4), (43, 3), (42 ^ (1 << 32), 3), (42, 3 + (1 << 8))):
        other = _device_mask(*shape, seed, call, p).double()
        near((keep == other).double().mean().item(), n, r, f"agreement with ({seed}, {call})")


@pytest.mark.parametrize("case_id", ["f32-D32-h2-seq2x1-L33-m9-nc", "f32-D64-h3-time1x3-L5-m4-c", "bf16-D64-h8-seq2x1-L65-m4-nc-gap"])
def test_mean_over_seeds_is_the_undropped_output(case_id, guard):
    """E[keep] s = 1: the mean of 256 dropout outputs (one seed each) is the undropped output within 6 sigma of the mean
    (sigma^2 = s^2 p (1 - p) sum_j w_j^2 v_j^2 / 256) plus the kernels' rounding."""
    case = [c for c in ATTN_CASES if _attn_id(c) == case_id][0]
    p, n_seeds = 0.3, 256
    call = _attn_setup(case, guard)
    acc_sum = torch.zeros_like(call.out, dtype=torch.float64)
    for seed in range(n_seeds):
        _run_dropout(call, seed * 7919 + 1, 0, p)
        acc_sum += call.out.double()
    mean = (acc_sum / n_seeds)[call.rows.reshape(-1)]
    q, k, v = call.operands()
    ref, acc, _ = _softmax64(q, k, v, call.causal, call.n_mem, call.kernel)
    S, H, L, D = q.shape
    s = dropout_scale(p)
    w = torch.einsum("shid,shjd->shij", q, k) * D ** -0.5
    if call.causal and L > 1:
        w = w.masked_fill(torch.ones((L, k.shape[2]), dtype=torch.bool, device=DEV).triu(call.n_mem + 1), -math.inf)
    w = w.softmax(-1)
    var = s * s * p * (1 - p) * torch.einsum("shij,shjd->shid", w * w, v * v)
    mean = mean.reshape(S, L, H, D).permute(0, 2, 1, 3)
    half_ulp = 2.0 ** -8 if call.code else 2.0 ** -24
    tol = 6 * (var / n_seeds).sqrt() + 4 * acc + 2 * half_ulp * (ref.abs() + var.sqrt()) + 1e-6 * ref.abs() + 1e-7
    assert ((mean - ref).abs() <= tol).all(), float(((mean - ref).abs() - tol).max())


# ------------------------------------------------------------------------------------------------------------------
# the tokenizer
# ------------------------------------------------------------------------------------------------------------------
def _models(name, p, dtype):
    g = load_golden(name)
    ms = []
    for pp in (0., p):
        m = build_product(dict(g["kwargs"], attn_dropout=pp), g["wseed"]).cuda()
        ms.append(m.bfloat16() if dtype == torch.bfloat16 else m)
    return g, ms


@pytest.mark.parametrize("name", ["mini", "cfg4"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_eval_outputs_are_those_of_attn_dropout_0(name, dtype, graphs):
    """Eval mode never drops: tokenize / decode_from_code_indices of attn_dropout=0.3 and 0 models with the same weights are
    bit-identical, and no random number is drawn."""
    g, (m0, m3) = _models(name, 0.3, dtype)
    video = golden_video(g).cuda().to(dtype)
    outs = []
    for m in (m0, m3):
        m.cuda_graphs = graphs
        rng = torch.get_rng_state()
        for _ in range(3 if graphs else 1):        # warm-up, capture, replay
            codes = m.tokenize(video)
            recon = m.decode_from_code_indices(codes)
        assert torch.equal(torch.get_rng_state(), rng)
        outs.append((codes, recon))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


SMALL64 = dict(image_size=64, init_dim=16, max_dim=64, codebook_size=1024, use_gan=False, perceptual_loss_weight=0.,
               layers=("residual", "compress_space", "attend_space", "compress_time", "attend_time"))


def _config(which):
    """(kwargs, video, torch seed of the step): the mini LFQ config (space attention L = 16, time attention L = 5), or one whose
    space attention has L = 1024 so that a bf16 step runs attention_mma_dropout_kernel.  The seeds leave every pre-sign value
    of the float64 oracle at least 2e-4 from 0 (3.4e-3 and 3.1e-4)."""
    from oracle import weights as W
    if which == "mini":
        g = load_golden("mini_train")
        return dict(g["kwargs"]), golden_video(g), 1234
    return dict(SMALL64), W.synth_video(1, 3, 1, 64, seed=77), 2


def _recording(monkeypatch):
    """Records the AttnDropout state of every dropout forward (its seed and how many attention calls it served)."""
    from magvit2_pytorch_b200 import video_tokenizer as VT
    seen = []

    class Rec(VT.AttnDropout):
        def __init__(self, *a):
            super().__init__(*a)
            seen.append(self)
    monkeypatch.setattr(VT, "AttnDropout", Rec)
    return seen


def _step(model, video, seed):
    model.train()
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(seed)
    total, bd = model(video, return_loss=True)
    total.backward()
    return total, bd


def _oracle_with_masks(monkeypatch, model_cpu, kw, seed, p):
    """float64 oracle whose k-th softmax attention applies the device mask of (seed, k), recording the pre-sign values."""
    from oracle import restated as R
    orc = build_oracle(model_cpu, kw, dtype=torch.float64)
    state = dict(calls=0, presign=None)
    s = dropout_scale(p)

    def softmax_attention(q, k, v, causal):
        b, h, i, d = q.shape
        j = k.shape[2]
        dots = torch.einsum("bhid,bhjd->bhij", q, k) * d ** -0.5
        if causal and i > 1:
            dots = dots.masked_fill(torch.ones((i, j), dtype=torch.bool).triu(j - i + 1), -torch.finfo(dots.dtype).max)
        keep = _device_mask(b, h, i, j - i, seed, state["calls"], p).cpu().to(q.dtype)
        state["calls"] += 1
        return torch.einsum("bhij,bhjd->bhid", dots.softmax(dim=-1) * keep * s, v)

    presign = R.lfq_presign

    def rec_presign(*a, **k):
        out = presign(*a, **k)
        state["presign"] = out.detach()
        return out

    monkeypatch.setattr(R, "softmax_attention", softmax_attention)
    monkeypatch.setattr(R, "lfq_presign", rec_presign)
    return orc, state


@pytest.mark.parametrize("which", ["mini", "space64"])
def test_training_gradients_vs_float64_oracle(monkeypatch, which):
    """fp32 train step at attn_dropout = 0.2 against the float64 oracle applying the same masks: loss and every parameter
    gradient; then the bf16 step under the same seed (same masks) agrees with fp32 as test_bf16_gradients_agree_with_fp32."""
    from oracle.make_train_golden import grad_digest
    from tests.test_oracle import grad_digest_close
    from torch.profiler import ProfilerActivity, profile
    p = 0.2
    kw, video, tseed = _config(which)
    kw = dict(kw, attn_dropout=p)
    seen = _recording(monkeypatch)
    cpu = build_product(kw, 0)
    model = build_product(kw, 0).cuda()
    total, bd = _step(model, video.cuda(), tseed)
    assert len(seen) == 1 and seen[0].calls == 2 * sum(1 for l in kw["layers"] if l in ("attend_space", "attend_time"))
    orc, state = _oracle_with_masks(monkeypatch, cpu, kw, seen[0].seed, p)
    for t in orc.sd.values():
        if t.is_floating_point():
            t.requires_grad_(True)
    out = orc.loss_forward(video.double(), train=True)
    assert state["calls"] == seen[0].calls
    margin = float(state["presign"].abs().min())
    assert margin > 2e-4, f"precondition: a pre-sign value {margin:.2e} near 0 could flip its code between fp32 and float64"
    ref = float(out["total_loss"].detach())
    assert abs(total.item() - ref) < 1e-4 * max(1.0, abs(ref)), (total.item(), ref)
    out["total_loss"].backward()
    named = dict(model.named_parameters())
    grads = {k: t.grad for k, t in orc.sd.items() if k in named and t.grad is not None and float(t.grad.abs().max()) > 0}
    gnorm = sum(float(g.norm()) ** 2 for g in grads.values()) ** 0.5
    worst = 0.0
    for k, g in grads.items():
        worst = max(worst, grad_digest_close(named[k].grad, grad_digest(g.float()), 5e-3, k, atol=1e-7 * gnorm))
    assert len(grads) >= 30, len(grads)
    print(f"{which}: {len(grads)} gradients vs float64, worst relative deviation {worst:.2e}, min |pre-sign| {margin:.2e}")

    # bf16 against fp32 on the reconstruction loss under the same seed
    kw0 = dict(kw, quantizer_aux_loss_weight=0.)
    m32 = build_product(kw0, 0).cuda()
    m16 = build_product(kw0, 0).cuda().bfloat16()
    t32, _ = _step(m32, video.cuda(), tseed)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t16, _ = _step(m16, video.cuda().bfloat16(), tseed)
        torch.cuda.synchronize()
    names = {_short(e.name).split("<")[0] for e in prof.events() if "attention" in e.name}
    if which == "space64":
        assert "attention_mma_dropout_kernel" in names, names
    assert abs(t16.float().item() - t32.item()) < 0.05 * abs(t32.item()) + 0.05

    def cosine(prefixes):
        num = da = db = 0.0
        for (k, a), (_, b) in zip(m32.named_parameters(), m16.named_parameters()):
            if a.grad is None or b.grad is None or not k.startswith(prefixes):
                continue
            ga, gb = a.grad.double().flatten(), b.grad.double().flatten()
            num += float(ga @ gb); da += float(ga @ ga); db += float(gb @ gb)
        return num / (da ** 0.5 * db ** 0.5)

    assert cosine(("decoder_layers", "conv_out", "quantizers.project_out")) > 0.95
    assert cosine(("encoder_layers", "conv_in", "quantizers.project_in")) > 0.5


def test_reproducible_from_torch_seed():
    """The same torch.manual_seed gives bit-identical losses and gradients, another seed changes them; a p = 0 step leaves
    torch's CPU generator untouched, a p > 0 step advances it."""
    kw, video, _ = _config("mini")
    video = video.cuda()
    runs = []
    for seed in (5, 5, 6):
        m = build_product(dict(kw, attn_dropout=0.2), 0).cuda()
        total, _ = _step(m, video, seed)
        runs.append((total.detach(), [q.grad.clone() for q in m.parameters() if q.grad is not None]))
    assert torch.equal(runs[0][0], runs[1][0]) and all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    assert not torch.equal(runs[0][0], runs[2][0])
    for p, moves in ((0., False), (0.2, True)):
        m = build_product(dict(kw, attn_dropout=p), 0).cuda().train()
        torch.manual_seed(9)
        rng = torch.get_rng_state()
        total, _ = m(video, return_loss=True)
        total.backward()
        assert torch.equal(torch.get_rng_state(), rng) != moves, p


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_no_grad_train_forward_drops(monkeypatch, graphs):
    """model.train(); model(v, return_recon=True) without gradients drops: it differs from eval, matches the reconstruction of
    the grad step under the same seed (same masks; the step runs the residual units unfused, hence allclose), and consecutive
    calls differ -- with cuda_graphs=True too, whose dropout forwards run outside the graphs."""
    from magvit2_pytorch_b200 import train as T
    kw, video, _ = _config("mini")
    video = video.cuda()
    m = build_product(dict(kw, attn_dropout=0.2), 0).cuda()
    m.cuda_graphs = graphs
    with torch.no_grad():
        ev = m.eval()(video, return_recon=True)
        m.train()
        torch.manual_seed(3)
        r = [m(video, return_recon=True) for _ in range(3)]
        torch.manual_seed(3)
        again = m(video, return_recon=True)
    assert torch.equal(r[0], again)
    assert not torch.equal(r[0], r[1]) and not torch.equal(r[1], r[2])
    assert (r[0] - ev).abs().max() > 1e-3
    if graphs:
        return
    got = {}
    fwd = T.TrainRunner.forward

    def rec(self, *a, **k):
        out = fwd(self, *a, **k)
        got["recon"] = out[0].detach().clone()
        return out
    monkeypatch.setattr(T.TrainRunner, "forward", rec)
    _step(m, video, 3)
    assert torch.allclose(got["recon"], r[0], rtol=1e-4, atol=1e-5), float((got["recon"] - r[0]).abs().max())
    assert (got["recon"] - r[1]).abs().max() > 10 * (got["recon"] - r[0]).abs().max()
