"""LFQ codebooks past 2^16 codes (MAGVIT-v2's 2^18): construction limits of the quantiser modules, and the bit-factorised
entropy gradient the device kernels implement (mv2_lfq_entropy_fact_backward), checked in float64 against autograd of the
dense clamped-entropy loss.  CPU only."""
import pytest
import torch

from magvit2_pytorch_b200 import modules as Mods

LFQ_KW = dict(entropy_loss_weight=0.1, commitment_loss_weight=1.0, diversity_gamma=2.5, soft_clamp_input_value=10.0)


@pytest.mark.parametrize("K,nc", [(2 ** 18, 1), (2 ** 20, 1), (2 ** 16, 2)], ids=["2^18", "2^20", "2x2^16"])
def test_lfq_large_codebook_constructs(K, nc):
    q = Mods.LFQ(64, K, num_codebooks=nc, **LFQ_KW)
    d = K.bit_length() - 1
    assert q.codebook_dim == d and q.num_codebooks == nc
    assert tuple(q.project_in.weight.shape) == (d * nc, 64)
    assert q.mask.tolist() == [2 ** i for i in range(d - 1, -1, -1)]


def test_quantiser_dims_limit():
    Mods.LFQ(64, 2 ** 16, num_codebooks=2, **LFQ_KW)                 # D = 32: the widest kernel instantiation
    with pytest.raises(NotImplementedError, match="32 projected dims"):
        Mods.LFQ(64, 2 ** 11, num_codebooks=3, **LFQ_KW)            # D = 33
    Mods.FSQ([8, 5, 5] * 8, 64)                                      # D = 24
    with pytest.raises(NotImplementedError, match="32 projected dims"):
        Mods.FSQ([2] * 11, 64, num_codebooks=3)


def _codebook(d):
    mask = 2 ** torch.arange(d - 1, -1, -1)
    return ((torch.arange(2 ** d)[:, None] & mask) != 0).double() * 2 - 1


def _h(x, eps=1e-5):
    return (-x * torch.log(x.clamp(min=eps))).sum(dim=-1)


def _factorised_grad(p, avg_global, inv_t, w_e, gamma, eps=1e-5):
    """The gradient the backward kernel computes, written out densely: prob from the per-bit sigmoids,
    c_tk = prob_tk (w_e/(N nc) h'(prob_tk) - w_e gamma/(N nc) h'(avg_global_k)),
    dp_ti = 2 tau (sum_k c_tk s_ki - tanh(2 tau p_ti) sum_k c_tk)."""
    N, nc, d = p.shape
    cb = _codebook(d)
    s = torch.sigmoid(4 * inv_t * p)                                                    # P(bit = +1), (N, nc, d)
    prob = torch.where(cb > 0, s[:, :, None, :], 1 - s[:, :, None, :]).prod(dim=-1)     # (N, nc, K)
    hp = lambda x: torch.where(x > eps, -(torch.log(x) + 1), torch.full_like(x, -torch.log(torch.tensor(eps, dtype=x.dtype)).item()))
    c = prob * (w_e / (N * nc) * hp(prob) - w_e * gamma / (N * nc) * hp(avg_global)[None])
    return 2 * inv_t * (torch.einsum("tck,kd->tcd", c, cb) - torch.tanh(2 * inv_t * p) * c.sum(dim=-1, keepdim=True))


@pytest.mark.parametrize("d,nc,inv_t", [(3, 1, 100.0), (3, 2, 1.0), (8, 1, 100.0), (8, 2, 1.0)])
def test_factorised_gradient_matches_dense_autograd(d, nc, inv_t):
    g = torch.Generator().manual_seed(d * 10 + nc)
    N, w_e, gamma = 37, 0.1, 2.5
    p = (torch.rand(N, nc, d, generator=g, dtype=torch.float64) * 2 - 1) * (0.05 if inv_t > 10 else 1.0)
    p[0] = 0                                               # a uniform token
    p[1] = torch.sign(p[1]) * (0.9 if inv_t > 10 else 5.0)   # a confident one: most codes under the clamp
    p.requires_grad_(True)
    # a cross-rank mean that differs from this rank's: another rank's tokens averaged in
    other = torch.softmax(torch.randn(nc, 2 ** d, generator=g, dtype=torch.float64) * 3, dim=-1)
    cb = _codebook(d)
    prob = (2 * inv_t * torch.einsum("tcd,kd->tck", p, cb)).softmax(dim=-1)
    avg_local = prob.mean(dim=0)
    avg_global = (avg_local.detach() + other) / 2
    assert (prob < 1e-5).any() and (prob > 1e-5).any()     # both sides of the clamp are exercised
    avg = avg_local + (avg_global - avg_local).detach()
    loss = w_e * (_h(prob).mean() - gamma * _h(avg).mean())
    want, = torch.autograd.grad(loss, p)
    got = _factorised_grad(p.detach(), avg_global, inv_t, w_e, gamma)
    assert torch.allclose(got, want, rtol=1e-9, atol=1e-12 * want.abs().max().item())
    # the product of per-bit sigmoids is the softmax over the codes
    s = torch.sigmoid(4 * inv_t * p.detach())
    prob_f = torch.where(cb > 0, s[:, :, None, :], 1 - s[:, :, None, :]).prod(dim=-1)
    assert torch.allclose(prob_f, prob.detach(), rtol=0, atol=1e-14)
