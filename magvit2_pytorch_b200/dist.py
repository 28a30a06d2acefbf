"""Multi-GPU plumbing for the VideoTokenizer path (SURVEY.md 8e): one process per GPU, torch.distributed (NCCL on
GPUs, gloo in the CPU tests) for the plumbing.

The eval forward is batch independent, so clips are simply sharded across ranks with NO data-path collective.
The only collective on the path is LFQ's training-mode batch-entropy term (SURVEY.md Appendix A.1 step 7; reached
from reference M:1705): every rank's mean code-probability vector ``avg_prob`` (num_codebooks x codebook_size fp32:
nc * 2^d * 4 bytes, 4 KiB at the README config, 1 MiB at MAGVIT-v2's 2^18 codes) is summed over ranks and divided by the
world size.  It is latency bound, so it is
issued on a side stream and overlaps whatever the caller runs next (the decoder).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of n clips owned by `rank` (first n % world ranks get one extra)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_clips(batch: torch.Tensor, rank: Optional[int] = None, world: Optional[int] = None) -> torch.Tensor:
    if rank is None or world is None:
        if dist.is_available() and dist.is_initialized():
            rank, world = dist.get_rank(), dist.get_world_size()
        else:
            rank, world = 0, 1
    lo, hi = shard_range(batch.shape[0], rank, world)
    return batch[lo:hi]


def allreduce_mean_(t: torch.Tensor, group=None, async_op: bool = False):
    """In-place cross-rank mean (SUM all-reduce then / world), as vector-quantize-pytorch's maybe_distributed_mean.
    No-op when torch.distributed is not initialised or world == 1.  Returns the work handle when async_op."""
    if not (dist.is_available() and dist.is_initialized()):
        return None
    world = dist.get_world_size(group)
    if world == 1:
        return None
    work = dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
    if async_op:
        return work, world
    t.div_(world)
    return None


def entropy_from_avg_prob(avg_prob: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """codebook (batch) entropy  sum_k -p_k log(clamp(p_k, eps))  (A.1 step 7)."""
    return (-avg_prob * torch.log(avg_prob.clamp(min=eps))).sum(dim=-1)


# codebook dims per codebook (d = log2(codebook_size)) of the LFQ training-mode terms: up to LFQ_DENSE_MAX_D the per-token
# softmax over all 2^d codes runs in shared memory (mv2_lfq_entropy_partials); above, the bit-factorised kernels take it
# (mv2_lfq_entropy_fact_*, d <= LFQ_TRAIN_MAX_D)
LFQ_DENSE_MAX_D = 12
LFQ_TRAIN_MAX_D = 20


def check_lfq_train_dim(d: int):
    if d > LFQ_TRAIN_MAX_D:
        raise NotImplementedError(f"LFQ training-mode losses take codebook_size <= 2^{LFQ_TRAIN_MAX_D} per codebook "
                                  f"(got 2^{d}); tokenize / decode take any size up to 32 projected dims")


class LfqBatchEntropy:
    """LFQ training-mode auxiliary terms on the GPU: per-rank partials (mv2_lfq_entropy_partials for d <= 12, the
    bit-factorised mv2_lfq_entropy_fact_partials for 12 < d <= 20), then the all-reduce of avg_prob (nc * 2^d * 4 bytes)
    on a side stream.  start() launches; finish() returns (per_sample_entropy, batch_entropy, commitment, aux_loss) as
    0-d tensors."""

    def __init__(self, engine, inv_temperature: float = 100.0, num_codebooks: int = 1):
        self.eng = engine
        self.nc = int(num_codebooks)
        self.inv_temperature = inv_temperature
        self.side = torch.cuda.Stream(device=engine.device)
        self._pending = None

    def start(self, presign: torch.Tensor, group=None):
        eng = self.eng
        N, D = presign.shape
        d = D // self.nc                 # presign is [N][num_codebooks][d]
        check_lfq_train_dim(d)
        K = 1 << d
        avg = torch.zeros(self.nc * K, device=presign.device, dtype=torch.float32)
        stats = torch.zeros(2, device=presign.device, dtype=torch.float32)
        ws = None
        if d > LFQ_DENSE_MAX_D:
            ws = torch.empty(eng.lib.mv2_lfq_entropy_fact_workspace_bytes(N, d, self.nc), device=presign.device, dtype=torch.uint8)
        self.side.wait_stream(torch.cuda.current_stream(eng.device))
        with torch.cuda.stream(self.side):
            st = C.c_void_p(self.side.cuda_stream)
            if ws is None:
                eng._call("mv2_lfq_entropy_partials", presign.data_ptr(), N, d, self.nc, float(self.inv_temperature), avg.data_ptr(),
                          stats.data_ptr(), stream=st)
            else:
                eng._call("mv2_lfq_entropy_fact_partials", presign.data_ptr(), N, d, self.nc, float(self.inv_temperature),
                          avg.data_ptr(), stats.data_ptr(), ws.data_ptr(), stream=st)
                ws.record_stream(self.side)
            avg.div_(N)                       # local mean code probability
            if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
                dist.all_reduce(avg, op=dist.ReduceOp.SUM, group=group)    # the one collective of the path (NCCL, nc * 2^d * 4 bytes)
        presign.record_stream(self.side)
        self._pending = (avg, stats, N, d)

    @property
    def avg_prob_sum(self) -> torch.Tensor:
        """[num_codebooks * K] SUM over ranks of the per-rank mean code probabilities of the pending start() (valid on the side
        stream; finish() orders the caller's stream after it)."""
        return self._pending[0]

    def finish(self, diversity_gamma=2.5, entropy_w=0.1, commit_w=1.0, group=None):
        """-> (per_sample_entropy, batch_entropy, commitment, aux_loss) as 0-d fp32 tensors (views of one 4-float result of
        mv2_lfq_aux_finalize).  `avg` holds the SUM over ranks of the per-rank mean code probabilities (start() divides by the
        local token count before the all-reduce, as the reference's maybe_distributed_mean does), so p = avg / world."""
        avg, stats, N, d = self._pending
        eng = self.eng
        torch.cuda.current_stream(eng.device).wait_stream(self.side)
        world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        out = torch.empty(4, device=avg.device, dtype=torch.float32)
        # avg is already a per-rank mean: "tokens_global" = number of ranks summed; per-rank terms use the local N
        eng._call("mv2_lfq_aux_finalize", avg.data_ptr(), stats.data_ptr(), d, self.nc, N, world, float(diversity_gamma),
                  float(entropy_w), float(commit_w), out.data_ptr())
        self._pending = None
        return out[0], out[1], out[2], out[3]
