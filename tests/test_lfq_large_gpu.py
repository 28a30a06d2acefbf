"""LFQ codebooks past 2^12 codes per codebook up to 2^20 (MAGVIT-v2's 2^18), and quantisers with 17 .. 32 projected dims:
the bit-factorised entropy kernels (mv2_lfq_entropy_fact_*) against a float64 dense enumeration of the codes, the wide
finalize, the wide quantiser forward / decode, the factorised training path against the dense torch one, and the reference
goldens mini_lfq18 / mini_mc16 (oracle/make_lfq_large_golden.py)."""
import ctypes as C

import pytest
import torch

from tests import test_simt_ops_gpu as S
from tests.test_oracle import grad_digest_close
from tests.util import build_product, golden_video, load_golden

pytestmark = pytest.mark.gpu

U = S.U
E_ARG = S.E_ARG
F32, BF16 = S.F32, S.BF16
LOG_INV_EPS = 11.512925464970229


def _ws(N, d, nc):
    n = S._lib().mv2_lfq_entropy_fact_workspace_bytes(N, d, nc)
    assert n > 0
    return torch.empty(n, device="cuda", dtype=torch.uint8)


def _fact_partials(p32, d, nc, inv_t):
    N = p32.shape[0]
    avg = torch.full((nc, 2 ** d), float("nan"), device="cuda", dtype=torch.float32)     # overwritten, not accumulated
    stats = torch.full((2,), float("nan"), device="cuda", dtype=torch.float32)
    S._ok(S._lib().mv2_lfq_entropy_fact_partials(p32.data_ptr(), N, d, nc, inv_t, avg.data_ptr(), stats.data_ptr(),
                                                 _ws(N, d, nc).data_ptr(), S._st()), "mv2_lfq_entropy_fact_partials")
    return avg, stats


def _fact_backward(p32, avg_global, d, nc, inv_t, cs, cb):
    N = p32.shape[0]
    gp = torch.full_like(p32, float("nan"))
    S._ok(S._lib().mv2_lfq_entropy_fact_backward(p32.data_ptr(), avg_global.data_ptr(), N, d, nc, inv_t, cs, cb, gp.data_ptr(),
                                                 _ws(N, d, nc).data_ptr(), S._st()), "mv2_lfq_entropy_fact_backward")
    return gp


def _codebook(d, device="cuda"):
    mask = 2 ** torch.arange(d - 1, -1, -1, device=device)
    return ((torch.arange(2 ** d, device=device)[:, None] & mask) != 0).double() * 2 - 1


def _dense64(p, d, inv_t, hga=None, cs=0.0, chunk=8):
    """float64 dense enumeration, chunked over tokens: (sum of clamped per-token entropies, un-normalised avg_prob (nc, K))
    and, with hga = coef_batch * h'(avg_global) (nc, K), the pre-sign gradient and its round-off scale per token."""
    N, nc, _ = p.shape
    cb = _codebook(d)
    ent, avg = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros((nc, 2 ** d), dtype=torch.float64, device="cuda")
    grad, cabs = torch.zeros_like(p), torch.zeros_like(p)
    for t0 in range(0, N, chunk):
        pc = p[t0:t0 + chunk]
        prob = (2 * inv_t * torch.einsum("tcd,kd->tck", pc, cb)).softmax(dim=-1)
        ent += (-prob * torch.log(prob.clamp(min=1e-5))).sum()
        avg += prob.sum(dim=0)
        if hga is not None:
            hp = torch.where(prob > 1e-5, -(torch.log(prob) + 1), torch.full_like(prob, LOG_INV_EPS))
            c = prob * (cs * hp - hga[None])
            tc = c.sum(dim=-1, keepdim=True)
            grad[t0:t0 + chunk] = 2 * inv_t * (torch.einsum("tck,kd->tcd", c, cb) - torch.tanh(2 * inv_t * pc) * tc)
            # magnitude of the terms before any cancellation: the scale of the kernel's round-off
            cabs[t0:t0 + chunk] = (prob * (cs * hp.abs() + hga.abs()[None] + cs)).sum(dim=-1, keepdim=True)
        del prob
    return ent, avg, grad, cabs


def _presign(N, nc, d, inv_t, g):
    # multiples of 2^-8 in [-1, 1] (the code logits are then exact in fp32), scaled down at inv_t = 100 so that the codes spread
    p = torch.randint(-256, 257, (N, nc, d), generator=g, device="cuda").double() / 256
    if inv_t > 10:
        p = p / 16
    p[0] = 0                                                   # uniform over the 2^d codes: no code above the clamp at d >= 17
    p[1] = torch.where(p[1] >= 0, 1.0, -1.0)                   # |4 tau p| = 400: sigma underflows to 0 for the other sign
    p[2, :, : d // 2] = 0.5                                    # half confident, half spread
    return p


FACT_CASES = [(12, 1, 45, 100.0), (12, 2, 37, 1.0), (13, 1, 37, 100.0), (13, 2, 41, 1.0), (16, 1, 37, 1.0), (16, 2, 35, 100.0),
              (18, 1, 37, 100.0), (18, 1, 35, 1.0), (20, 1, 19, 100.0)]


@pytest.mark.parametrize("d,nc,N,inv_t", FACT_CASES, ids=[f"d{c[0]}-nc{c[1]}-N{c[2]}-it{c[3]:g}" for c in FACT_CASES])
def test_fact_partials_and_backward_vs_float64(d, nc, N, inv_t):
    g = S._gen(d * 1000 + nc * 100 + N)
    p = _presign(N, nc, d, inv_t, g)
    p32 = p.float().contiguous()
    avg, stats = _fact_partials(p32, d, nc, inv_t)
    # a cross-rank mean that differs from the local one
    other = torch.softmax(torch.randn((nc, 2 ** d), generator=g, device="cuda", dtype=torch.float64) * 4, dim=-1)
    w_e, gamma = 0.1, 2.5
    cs, cbt = w_e / (N * nc), w_e * gamma / (N * nc)
    ent, prob_sum, _, _ = _dense64(p, d, inv_t)
    avg_global = ((prob_sum / N + other) / 2).float().contiguous()
    a64 = avg_global.double()
    hga = cbt * torch.where(a64 > 1e-5, -(torch.log(a64) + 1), torch.full_like(a64, LOG_INV_EPS))
    _, _, grad, cabs = _dense64(p, d, inv_t, hga, cs)
    # partials: each prob is a product of d fp32 sigmoids (~3 ulp each); per thread 32-token x 16-code fp32 sums, then fp64
    rel = (6 * d + 600) * U
    tol0 = rel * (ent.item() + N * nc)
    assert abs(stats[0].item() - ent.item()) <= tol0, (stats[0].item(), ent.item())
    q = torch.where(p > 0, torch.ones_like(p), -torch.ones_like(p))
    com = ((p - q) ** 2).sum().item()
    assert abs(stats[1].item() - com) <= 8 * U * com
    assert ((avg.double() - prob_sum).abs() <= rel * prob_sum + 1e-37 * N).all()
    # the bound rejects the result with one token (the uniform one) left out
    ent_wrong, prob_wrong, _, _ = _dense64(p[1:], d, inv_t)
    assert abs(stats[0].item() - ent_wrong.item()) > tol0
    assert not ((avg.double() - prob_wrong).abs() <= rel * prob_wrong + 1e-37 * N).all()
    # backward: c_k to ~(2d + 30) ulp (sigmoid products, __logf, coefficients), sums over 2^d codes in fp32 per lane and warp tree
    gp = _fact_backward(p32, avg_global, d, nc, inv_t, cs, cbt)
    relg = (2 * d + 30 + 2 ** max(d - 10, 0) + 64) * U
    bound = 2 * inv_t * relg * 2 * cabs + 4 * U * grad.abs() + 1e-30
    excess = ((gp.double() - grad).abs() - bound).max().item()
    assert excess <= 0, excess
    # ... and rejects the gradient without the batch-entropy term
    _, _, grad_wrong, _ = _dense64(p, d, inv_t, torch.zeros_like(hga), cs)
    assert ((gp.double() - grad_wrong).abs() - bound).max().item() > 0
    # bit-identical across runs
    avg2, stats2 = _fact_partials(p32, d, nc, inv_t)
    gp2 = _fact_backward(p32, avg_global, d, nc, inv_t, cs, cbt)
    assert torch.equal(avg, avg2) and torch.equal(stats, stats2) and torch.equal(gp, gp2)


@pytest.mark.parametrize("nc,inv_t", [(1, 100.0), (2, 1.0)])
def test_fact_partials_agree_with_the_shared_memory_kernel_at_d12(nc, inv_t):
    g = S._gen(12 + nc)
    p32 = _presign(131, nc, 12, inv_t, g).float().contiguous()
    avg, stats = _fact_partials(p32, 12, nc, inv_t)
    avg_s, stats_s = S._entropy_run(p32.double(), 12, nc, inv_t)
    assert torch.allclose(avg, avg_s, rtol=2e-4, atol=1e-9)
    assert torch.allclose(stats, stats_s, rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("d,nc", [(16, 1), (13, 2), (20, 1)])
def test_wide_finalize_world_size_two(d, nc):
    """Two halves of the tokens with their avg_prob summed, as the cross-rank all-reduce does, reproduce the batch entropy of
    all tokens; the per-rank terms are the first half's."""
    g = S._gen(d + 7 * nc)
    N, inv_t = 64, 100.0
    p = _presign(N, nc, d, inv_t, g)
    h = N // 2
    a0, s0 = _fact_partials(p[:h].float().contiguous(), d, nc, inv_t)
    a1, _ = _fact_partials(p[h:].float().contiguous(), d, nc, inv_t)
    out4, asum = torch.empty(4, device="cuda", dtype=torch.float32), (a0 + a1).contiguous()
    S._ok(S._lib().mv2_lfq_aux_finalize(asum.data_ptr(), s0.data_ptr(), d, nc, h, 2 * h, 2.5, 0.1, 1.0, out4.data_ptr(), S._st()),
          "mv2_lfq_aux_finalize")
    ent0, _, _, _ = _dense64(p[:h], d, inv_t)
    _, prob_all, _, _ = _dense64(p, d, inv_t)
    pa = prob_all / N
    be = (-pa * torch.log(pa.clamp(min=1e-5))).sum(dim=-1).mean().item()
    ps = ent0.item() / (h * nc)
    q = torch.where(p[:h] > 0, torch.ones_like(p[:h]), -torch.ones_like(p[:h]))
    cm = ((p[:h] - q) ** 2).mean().item()
    want = [ps, be, cm, (ps - 2.5 * be) * 0.1 + cm]
    got = out4.cpu().tolist()
    for k in range(4):
        assert abs(got[k] - want[k]) <= 1e-4 * max(1.0, abs(want[k])), (k, got, want)


def test_new_entry_points_reject_out_of_range_arguments():
    lib = S._lib()
    st = S._st()
    buf = torch.zeros(1 << 16, device="cuda")
    p = buf.data_ptr()
    assert lib.mv2_lfq_entropy_fact_workspace_bytes(8, 21, 1) == 0
    assert lib.mv2_lfq_entropy_fact_partials(p, 8, 21, 1, 100.0, p, p, p, st) == E_ARG                  # d > 20
    assert lib.mv2_lfq_entropy_fact_backward(p, p, 8, 21, 1, 100.0, 0.1, 0.1, p, p, st) == E_ARG
    assert lib.mv2_lfq_entropy_fact_partials(p, 8, 17, 2, 100.0, p, p, p, st) == E_ARG                  # D = 34
    assert lib.mv2_lfq_entropy_fact_partials(p, 8, 0, 1, 100.0, p, p, p, st) == E_ARG
    assert lib.mv2_lfq_entropy_fact_partials(p, 8, 8, 1, 100.0, p, p, None, st) == E_ARG                # no workspace
    assert lib.mv2_lfq_aux_finalize(p, p, 21, 1, 8, 8, 2.5, 0.1, 1.0, p, st) == E_ARG
    assert lib.mv2_lfq_forward(p, F32, 8, 16, 11, 3, p, p, p, p, 10.0, 0, p, p, p, st) == E_ARG          # D = 33
    assert lib.mv2_lfq_decode(p, 1, 8, 16, 33, 1, p, p, p, F32, st) == E_ARG
    lv = (C.c_int32 * 11)(*([2] * 11))
    assert lib.mv2_fsq_forward(p, F32, 8, 16, 11, 3, lv, p, p, p, p, None, None, None, st) == E_ARG
    assert lib.mv2_fsq_decode(p, 0, 8, 16, 11, 3, lv, p, p, p, F32, st) == E_ARG


# the quantiser forward / decode on the wide (17 .. 32 projected dims) instantiation, with the checks of test_simt_ops_gpu
WIDE_LFQ_CASES = [(F32, 17, 1, 0, 10.0, 0, 72), (BF16, 18, 1, 1, 10.0, 1, 40), (F32, 16, 2, 1, 10.0, 0, 136),
                  (BF16, 8, 4, 0, 0.0, 0, 40), (F32, 31, 1, 0, 10.0, 1, 40)]


@pytest.mark.parametrize("code,d,nc,sph,clamp,zb,C_", WIDE_LFQ_CASES,
                         ids=[f"{'bf16' if c[0] else 'f32'}-{c[1]}x{c[2]}-sph{c[3]}" for c in WIDE_LFQ_CASES])
def test_lfq_wide(code, d, nc, sph, clamp, zb, C_):
    S.test_lfq(code, d, nc, sph, clamp, zb, C_)


@pytest.mark.parametrize("code", [F32, BF16], ids=["f32", "bf16"])
def test_fsq_wide(code):
    S.test_fsq(code, [8, 5, 5, 5], 6)                      # D = 24


# ------------------------------------------------------------------------------------------------------------------
# the training path: factorised autograd Function against the dense torch formulation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,nc,sph", [(13, 1, False), (13, 2, True), (14, 1, True), (14, 2, False)])
def test_lfq_train_factorised_matches_dense(d, nc, sph, monkeypatch):
    from magvit2_pytorch_b200 import modules as Mods
    from magvit2_pytorch_b200 import train as T
    torch.manual_seed(d * 10 + nc)
    qz = Mods.LFQ(48, 2 ** d, entropy_loss_weight=0.1, commitment_loss_weight=0.25, diversity_gamma=2.5, soft_clamp_input_value=10.0,
                  num_codebooks=nc, spherical=sph).cuda()
    x = torch.randn(2, 3, 7, 5, 48, device="cuda") * 0.05
    with torch.no_grad():
        qz.project_in.weight.mul_(0.5 if sph else 0.05)
    other = torch.softmax(torch.randn(nc, 2 ** d, device="cuda") * 3, dim=-1)

    def run():
        x_ = x.clone().requires_grad_(True)
        with torch.no_grad():      # this rank's mean code probability, averaged with another rank's
            p = F_presign(x_, qz, d, nc)
            cb = _codebook(d).float()
            avg_local = (200 * torch.einsum("tcd,kd->tck", p, cb)).softmax(dim=-1).mean(dim=0)
            avg_global = ((avg_local + other) / 2).reshape(-1)
        out, aux = T._lfq_train(x_, qz, avg_global)
        gx, gw = torch.autograd.grad(aux, [x_, qz.project_in.weight])
        return aux.detach(), gx, gw

    aux_f, gx_f, gw_f = run()
    monkeypatch.setattr(T, "LFQ_DENSE_MAX_D", 99)
    aux_d, gx_d, gw_d = run()
    assert abs(aux_f.item() - aux_d.item()) <= 2e-5 * max(1.0, abs(aux_d.item())), (aux_f.item(), aux_d.item())
    for a, b in ((gx_f, gx_d), (gw_f, gw_d)):
        assert (a - b).abs().max().item() <= 2e-3 * b.abs().max().item() + 1e-9, ((a - b).abs().max().item(), b.abs().max().item())


def F_presign(x, qz, d, nc):
    import torch.nn.functional as F
    p = F.linear(x, qz.project_in.weight, qz.project_in.bias)
    p = (p / 10.).tanh() * 10.
    p = p.reshape(-1, nc, d)
    return F.normalize(p, dim=-1).float() if qz.spherical else p.float()


# ------------------------------------------------------------------------------------------------------------------
# reference goldens
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["mini_lfq18", "mini_mc16"])
def test_large_codebook_codes_and_round_trip_vs_reference(name):
    g = load_golden(name)
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    video = golden_video(g).cuda()
    codes = model.tokenize(video)
    assert codes.dtype == torch.int64 and codes.shape == g["codes"].shape
    mism = codes.cpu() != g["codes"]
    margin = g["presign"].reshape(*g["codes"].shape, -1).abs().min(dim=-1).values      # per (token, codebook)
    assert (margin[mism].max().item() if mism.any() else 0.0) < 1e-5, margin[mism]
    recon = model.decode_from_code_indices(codes)
    with torch.no_grad():
        recon_fwd = model(video, return_recon=True)
    assert torch.equal(recon, recon_fwd)
    if not mism.any():
        assert (recon.cpu() - g["recon"]).abs().max().item() < 1e-3


@pytest.mark.parametrize("name", ["mini_lfq18_train", "mini_mc16_train"])
def test_large_codebook_losses_and_gradients_vs_reference_golden(name):
    g = load_golden(name)
    gt = g["train"]
    model = build_product(g["kwargs"], g["wseed"]).cuda()
    model.train()
    total, bd = model(golden_video(g).cuda(), return_loss=True)
    total.backward()
    assert abs(total.item() - gt["total_loss"].item()) < 1e-5
    assert abs(bd.recon_loss.item() - gt["recon_loss"].item()) < 1e-5
    assert abs(float(bd.lfq_aux_loss.detach()) - float(gt["aux"])) < 1e-5
    ps, be, cm = bd.quantizer_loss_breakdown
    for got, k in ((ps, "per_sample_entropy"), (be, "batch_entropy"), (cm, "commitment")):
        assert abs(got.item() - gt[k].item()) < 1e-5, k
    named = dict(model.named_parameters())
    gnorm = sum(d["norm"] ** 2 for d in gt["grads"].values() if d is not None) ** 0.5
    worst, checked = 0.0, 0
    for k, dg in gt["grads"].items():
        if k not in named:
            continue
        p = named[k]
        if dg is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        assert p.grad is not None, k
        worst = max(worst, grad_digest_close(p.grad, dg, 5e-3, k, atol=1e-7 * gnorm))
        checked += 1
    assert checked >= 50, checked
    print(f"{name}: {checked} parameter gradients checked, worst relative deviation vs the reference {worst:.2e}")


def test_bf16_train_step_at_2_18_codes():
    g = load_golden("mini_lfq18_train")
    model = build_product(g["kwargs"], g["wseed"]).cuda().bfloat16()
    model.train()
    total, bd = model(golden_video(g).cuda().bfloat16(), return_loss=True)
    total.backward()
    assert torch.isfinite(total).item()
    assert all(torch.isfinite(t).item() for t in bd.quantizer_loss_breakdown)
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert len(grads) >= 50 and all(torch.isfinite(gr).all().item() for gr in grads)
    assert model.quantizers.project_in.weight.grad.abs().max().item() > 0


def test_train_mode_rejects_codebooks_past_2_20():
    kw = dict(load_golden("mini_lfq18_train")["kwargs"], codebook_size=2 ** 21)       # use_gan=False, perceptual_loss_weight=0
    model = build_product(kw, 0).cuda()
    video = golden_video(load_golden("mini_lfq18")).cuda()
    codes = model.tokenize(video)                           # inference takes it
    assert int(codes.max()) < 2 ** 21
    with pytest.raises(NotImplementedError, match="2\\^20"):
        model.lfq_loss_breakdown(video)
    model.train()
    with pytest.raises(NotImplementedError, match="2\\^20"):
        model(video, return_loss=True)
