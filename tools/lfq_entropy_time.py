"""Times LFQ's training-mode entropy terms at the README token count (4 clips -> 5120 latent tokens, one codebook) for
codebook sizes 2^10 (the shared-memory softmax kernel, mv2_lfq_entropy_partials) and 2^14, 2^16, 2^18 (the bit-factorised
kernels, mv2_lfq_entropy_fact_*): forward partials + finalize, and the backward of the entropy terms to the pre-sign
values.  Also times the dense torch formulation of the same loss (the (tokens, nc, 2^d) softmax of train._lfq_train's
d <= 12 path, forward + autograd backward) and records its peak memory, where it fits.

Device events after a warm-up; prints the card's name and power limit with the numbers.

    python tools/lfq_entropy_time.py [--tokens 5120] [--iters 10]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from magvit2_pytorch_b200._lib import check, load  # noqa: E402
from tools.gan_step_time import _card, _time  # noqa: E402

INV_T, GAMMA, W_E = 100.0, 2.5, 0.1


def _dense_loss(p, avg_global, d):
    """train._lfq_train's dense entropy block on pre-sign values p (N, 1, d)."""
    mask = 2 ** torch.arange(d - 1, -1, -1, device=p.device)
    cb = ((torch.arange(2 ** d, device=p.device)[:, None] & mask) != 0).float() * 2 - 1
    prob = (2 * INV_T * torch.einsum("tcd,kd->tck", p, cb)).softmax(dim=-1)
    h = lambda x: (-x * torch.log(x.clamp(min=1e-5))).sum(dim=-1)
    avg_local = prob.mean(dim=0)
    avg = avg_local + (avg_global.reshape(1, -1) - avg_local).detach()
    return (h(prob).mean() - GAMMA * h(avg).mean()) * W_E


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=5120)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: timings are only taken on the GPU")
    lib = load()
    N, nc = args.tokens, 1
    g = torch.Generator(device="cuda").manual_seed(0)
    print(dict(card=_card(), tokens=N, num_codebooks=nc, inv_temperature=INV_T))
    for d in (10, 14, 16, 18):
        K = 1 << d
        # spherical-like pre-sign values: |p| ~ d^-1/2, so the 2 tau <p, c> logits spread over tens
        p = (torch.randn((N, nc, d), generator=g, device="cuda") * d ** -0.5).contiguous()
        avg = torch.zeros(nc * K, device="cuda")
        stats = torch.zeros(2, device="cuda")
        out4 = torch.empty(4, device="cuda")
        gp = torch.empty_like(p)
        st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
        fact = d > 12
        ws = torch.empty(max(1, lib.mv2_lfq_entropy_fact_workspace_bytes(N, d, nc)), device="cuda", dtype=torch.uint8)

        def partials():
            if fact:
                check(lib.mv2_lfq_entropy_fact_partials(p.data_ptr(), N, d, nc, INV_T, avg.data_ptr(), stats.data_ptr(), ws.data_ptr(), st()),
                      "mv2_lfq_entropy_fact_partials")
            else:
                avg.zero_()
                stats.zero_()
                check(lib.mv2_lfq_entropy_partials(p.data_ptr(), N, d, nc, INV_T, avg.data_ptr(), stats.data_ptr(), st()),
                      "mv2_lfq_entropy_partials")

        def finalize():
            check(lib.mv2_lfq_aux_finalize(avg.data_ptr(), stats.data_ptr(), d, nc, N, 1, GAMMA, W_E, 1.0, out4.data_ptr(), st()),
                  "mv2_lfq_aux_finalize")

        def backward():
            check(lib.mv2_lfq_entropy_fact_backward(p.data_ptr(), avg.data_ptr(), N, d, nc, INV_T, W_E / (N * nc),
                                                    W_E * GAMMA / (N * nc), gp.data_ptr(), ws.data_ptr(), st()),
                  "mv2_lfq_entropy_fact_backward")

        row = dict(d=d, codebook_size=K, path="factorised" if fact else "shared-memory softmax")
        row["partials_ms"] = round(_time(partials, args.iters), 4)
        partials()
        avg.div_(N)
        row["finalize_ms"] = round(_time(finalize, args.iters), 4)
        if fact:
            row["backward_ms"] = round(_time(backward, args.iters), 4)
        # the dense torch formulation (forward + autograd backward), where it fits
        avg_global = avg.clone()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        pd = p.clone().requires_grad_(True)

        def dense():
            loss = _dense_loss(pd, avg_global, d)
            torch.autograd.grad(loss, pd)

        try:
            row["dense_torch_fwd_bwd_ms"] = round(_time(dense, max(2, args.iters // 5), warmup=1), 3)
            row["dense_torch_peak_GB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)
        except torch.cuda.OutOfMemoryError:
            row["dense_torch_fwd_bwd_ms"] = "out of memory"
        del pd
        torch.cuda.empty_cache()
        row["pairs_per_pass_G"] = round(N * nc * K / 1e9, 3)
        print(row)


if __name__ == "__main__":
    main()
