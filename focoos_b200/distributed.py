"""Multi-GPU plumbing for the inference hot path: "replicas only".

Images are independent units, so the path shards with NO data-path collective (SURVEY.md §8e): one process per GPU,
each with a full model replica, the batch split evenly on the host.  `torch.distributed` (NCCL on GPUs, gloo in the CPU
tests) is used only to agree on the wall/devices timing (barrier + max over ranks), to gather per-rank detection
counts for reporting, and to combine the evaluators' state (box-AP records, confusion matrix) on rank 0.  Mirrors the role of `focoos/utils/distributed/{dist,comm}.py` for inference
(`comm.get_rank/get_world_size/synchronize/all_gather`), minus DDP (fine-tuning is a later round).
"""
from __future__ import annotations

import os
from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def get_rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def get_world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def init_from_env(backend: str = "nccl", device: torch.device | None = None) -> Tuple[int, int, int]:
    """Initialise the default group from torchrun's env (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*). Returns (rank, local_rank, world)."""
    rank, local_rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if world > 1 and not dist.is_initialized():
        kw = {"device_id": device} if (backend == "nccl" and device is not None) else {}
        dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    return rank, local_rank, world


def shard_range(n_items: int, rank: int | None = None, world: int | None = None) -> Tuple[int, int]:
    """Contiguous, balanced [begin, end) slice of `n_items` independent units for this rank (first `n % world` ranks get one more)."""
    rank = get_rank() if rank is None else rank
    world = get_world_size() if world is None else world
    base, extra = divmod(n_items, world)
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


def shard_list(items: Sequence, rank: int | None = None, world: int | None = None) -> List:
    b, e = shard_range(len(items), rank, world)
    return list(items[b:e])


def synchronize():
    if get_world_size() > 1:
        dist.barrier()


def max_over_ranks(value: float, device: torch.device | str = "cpu") -> float:
    """Multi-GPU timings are reported as the max over ranks (never the mean, never wall clock of rank 0)."""
    if get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_counts(count: int, device: torch.device | str = "cpu") -> List[int]:
    """all_gather of one integer per rank (e.g. images processed) so rank 0 can report whole-job totals."""
    if get_world_size() == 1:
        return [int(count)]
    t = torch.tensor([int(count)], dtype=torch.int64, device=device)
    out = [torch.zeros_like(t) for _ in range(get_world_size())]
    dist.all_gather(out, t)
    return [int(o.item()) for o in out]


def collective_device() -> torch.device:
    """where the default group's collectives take their tensors: the current GPU under NCCL, the host otherwise (gloo)"""
    if get_world_size() > 1 and dist.get_backend() == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def all_gather_rows(t: torch.Tensor) -> List[torch.Tensor]:
    """all_gather of a [n, ...] tensor whose n differs between ranks (evaluation records): padded to the largest n, trimmed after -> one tensor per rank,
    in rank order, on collective_device()"""
    t = t.to(collective_device())
    if get_world_size() == 1:
        return [t]
    n = gather_counts(t.shape[0], t.device)
    pad = t.new_zeros((max(n),) + tuple(t.shape[1:]))
    pad[: t.shape[0]] = t
    out = [torch.empty_like(pad) for _ in n]
    dist.all_gather(out, pad)
    return [o[:k] for o, k in zip(out, n)]


def all_reduce_sum(t: torch.Tensor) -> torch.Tensor:
    """SUM over the ranks of a copy of `t`, on collective_device() (`t` itself is left as it is)"""
    t = t.to(collective_device(), copy=True)
    if get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t
