"""Multi-GPU plumbing for the forward path: batch sharding and max-over-ranks timing.

The reference distributes with HF Trainer + DeepSpeed ZeRO-3 (train.sh:14-16, configs/deepspeed_config.json); the
forward itself is embarrassingly parallel over samples (SURVEY.md §8e), so the GPU path runs one full replica per
rank on a contiguous slice of the global batch with NO collective on the data path.  The only cross-rank traffic is
the scalar reduction used for timing / loss reporting.
"""
from __future__ import annotations

from typing import Tuple

import torch
import torch.distributed as dist


def shard_range(global_batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of the global batch owned by `rank` (sizes differ by at most one)."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world {world}")
    base, rem = divmod(global_batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_inputs(inputs: dict, rank: int, world: int) -> dict:
    """Slice every batched tensor of a reference-style `inputs` dict (llm_trainer.py:366-381) along dim 0."""
    B = inputs["input_ids"].shape[0]
    lo, hi = shard_range(B, rank, world)
    out = {}
    for k, v in inputs.items():
        out[k] = v[lo:hi] if isinstance(v, torch.Tensor) and v.dim() > 0 and v.shape[0] == B else v
    return out


def max_over_ranks(value: float, device=None) -> float:
    """MAX all-reduce of a scalar (elapsed milliseconds) over the default process group; identity without one."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def weighted_mean_loss(loss_sum: float, n_valid: int, device=None) -> float:
    """Global mean CE over all ranks' valid tokens (local means are NOT averaged: they are weighted by token count)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return loss_sum / max(n_valid, 1)
    t = torch.tensor([loss_sum, float(n_valid)], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t[0] / t[1].clamp_min(1.0))


# ---------------------------------------------------------------------------------------------------- gradient all-reduce
_NCCL_READY = False


def init_nccl(device=None) -> bool:
    """Create the kernel library's own NCCL communicator for the default torch.distributed group (one process per GPU):
    rank 0 draws the unique id (mm_nccl_unique_id) and ships it through torch.distributed's broadcast (plumbing), every
    rank calls mm_nccl_init.  Returns True when the communicator is up."""
    global _NCCL_READY
    if _NCCL_READY:
        return True
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return False
    import ctypes as C

    from . import _lib

    lib = _lib.load()
    world, rank = dist.get_world_size(), dist.get_rank()
    buf = (C.c_ubyte * 128)()
    if rank == 0:
        rc = lib.mm_nccl_unique_id(buf)
        if rc != 0:
            raise RuntimeError(f"mm_nccl_unique_id failed: {_lib.last_error()}")
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    t = torch.tensor(list(buf), dtype=torch.uint8, device=dev)
    dist.broadcast(t, src=0)
    ids = (C.c_ubyte * 128)(*t.cpu().tolist())
    with torch.cuda.device(dev):
        rc = lib.mm_nccl_init(ids, world, rank)
    if rc != 0:
        raise RuntimeError(f"mm_nccl_init failed: {_lib.last_error()}")
    _NCCL_READY = True
    return True


def nccl_allreduce_(t: torch.Tensor, average: bool = True) -> None:
    """In-place all-reduce of a contiguous bf16 / fp16 / fp32 CUDA tensor on torch's CURRENT stream through
    mm_nccl_allreduce."""
    from . import _lib

    codes = {torch.bfloat16: 0, torch.float32: 1, torch.float16: 2}
    assert _NCCL_READY and t.is_cuda and t.is_contiguous() and t.dtype in codes
    rc = _lib.load().mm_nccl_allreduce(t.data_ptr(), t.numel(), codes[t.dtype], int(average),
                                       torch.cuda.current_stream().cuda_stream)
    if rc != 0:
        raise RuntimeError(f"mm_nccl_allreduce failed: {_lib.last_error()}")


def destroy_nccl() -> None:
    global _NCCL_READY
    if _NCCL_READY:
        from . import _lib

        _lib.load().mm_nccl_destroy()
        _NCCL_READY = False
