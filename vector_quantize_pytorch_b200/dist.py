"""Multi-GPU plumbing of the EMA update (SURVEY.md §8e).

The path shards naturally: tokens are independent given the codebook, so the batch is split over the
ranks (one process per GPU) and the only exchange is the SUM of the per-rank batch statistics.  The
reference issues two all-reduces per codebook per stage (vector_quantize_pytorch.py:603, :607); here
every codebook touched by a forward writes its statistics into ONE packed fp32 buffer
`[cluster_size (K, padded to 4) | embed_sum (K x D)]*` and a single `all_reduce` (NCCL over NVLink on
GPUs, gloo in the CPU tests) covers them all.  After the reduction every rank applies the identical EMA
kernel to identical numbers, so the replicas' codebooks stay bit-identical.
"""
from __future__ import annotations

import torch
import torch.distributed as distributed

from ._C import lib


def is_distributed() -> bool:
    return distributed.is_available() and distributed.is_initialized() and distributed.get_world_size() > 1


def stats_layout(codebooks: list[tuple[int, int]]) -> tuple[list[int], list[int], int]:
    """codebooks: [(K, D), ...] -> (offsets, sizes, total) in floats of the packed statistics buffer."""
    sizes = [int(lib.vqb_stats_floats(K, D)) for K, D in codebooks]
    offsets, pos = [], 0
    for s in sizes:
        offsets.append(pos)
        pos += s
    return offsets, sizes, pos


def split_stats(stats: torch.Tensor, K: int, D: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Views (cluster_size (K,), embed_sum (K, D)) into one codebook's slice of the packed buffer."""
    off = int(lib.vqb_stats_offset(K))
    return stats[:K], stats[off:off + K * D].view(K, D)


def allreduce_packed(packed: torch.Tensor, group=None) -> torch.Tensor:
    """In-place SUM over ranks of the packed statistics (no-op outside a process group)."""
    if is_distributed():
        distributed.all_reduce(packed, op=distributed.ReduceOp.SUM, group=group)
    return packed


class PeerReducer:
    """The packed statistics of one module in SYMMETRIC memory (torch.distributed._symmetric_memory): every rank's
    buffer is mapped into every peer's address space over NVLink, so the EMA kernels sum all ranks' statistics with
    peer loads after one cross-GPU barrier kernel (csrc/vq_peer.cu) — no collective call, nothing between the
    statistics kernels and the EMA kernels that a CUDA graph could not hold.

    Two buffers alternate by step parity (see the protocol in vq_peer.cu).  `create` returns None when symmetric memory
    is unavailable (CPU / gloo group, no P2P): the callers then fall back to ONE NCCL all-reduce of the packed buffer."""

    def __init__(self, numel, device, hdls, bufs, flags, flags_hdl):
        import ctypes
        self.numel, self.device = numel, device
        self.world, self.rank = hdls[0].world_size, hdls[0].rank
        self.bufs = bufs
        self._hdls, self._flags, self._flags_hdl = hdls, flags, flags_hdl   # keep the mappings alive
        PtrArr = ctypes.c_void_p * self.world
        self.stats_ptrs = [PtrArr(*[int(p) for p in h.buffer_ptrs]) for h in hdls]
        self.flag_ptrs = PtrArr(*[int(p) for p in flags_hdl.buffer_ptrs])
        self.epoch = torch.zeros((1,), dtype=torch.int32, device=device)
        self.step = 0

    @staticmethod
    def create(numel: int, device, group=None):
        import os
        if not is_distributed() or torch.device(device).type != "cuda" or os.environ.get("VQB_NO_PEER"):
            return None
        if distributed.get_backend(group) != "nccl":
            return None
        try:
            import torch.distributed._symmetric_memory as symm
            group = group if group is not None else distributed.group.WORLD
            numel = (int(numel) + 3) // 4 * 4
            bufs = [symm.empty((numel,), dtype=torch.float32, device=device) for _ in range(2)]
            hdls = [symm.rendezvous(b, group) for b in bufs]
            flags = symm.empty((64,), dtype=torch.int32, device=device)
            flags.zero_()
            flags_hdl = symm.rendezvous(flags, group)
            if hdls[0].world_size > 16:
                return None
            pr = PeerReducer(numel, torch.device(device), hdls, bufs, flags, flags_hdl)
            torch.cuda.synchronize(device)
            distributed.barrier(group)   # every rank's flags are zero before anybody posts into them
            return pr
        except Exception as ex:  # noqa: BLE001 — any rendezvous / capability problem: NCCL path
            import warnings
            warnings.warn(f"vqb200: symmetric memory unavailable ({ex!r}); the EMA statistics use ncclAllReduce instead")
            return None

    def next_buffer(self) -> tuple[torch.Tensor, "ctypes.Array"]:
        """(this rank's statistics buffer for the coming step, host array of every rank's pointer to it)."""
        i = self.step & 1
        self.step += 1
        return self.bufs[i], self.stats_ptrs[i]

    def barrier(self):
        from . import ops
        ops.peer_barrier(self)


def shard_rows(n_rows: int, world: int, rank: int) -> tuple[int, int]:
    """Contiguous, balanced split of the batch rows over the ranks."""
    base, rem = divmod(n_rows, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)
