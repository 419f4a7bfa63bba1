"""Data-parallel plumbing for the LoRA step (one process per GPU, torch.distributed).

The path shards by data only: every rank holds a full replica, processes its own
image(s) and the single exchange is a SUM all-reduce of the flat LoRA-gradient buffer; the 1/world
average is folded into the fused clip+AdamW kernel. Replaces what the reference gets from
accelerate -> DDP (training_scripts/train_lora_dreambooth.py:744-757, 877)."""
from typing import List

import torch


def world_info():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_indices(n_items: int, rank: int, world: int, drop_last: bool = False) -> List[int]:
    """Round-robin dataset sharding (accelerate's prepared DataLoader semantics: rank r takes
    items r, r+world, ...). Without drop_last the tail is padded by wrapping so that every rank
    runs the same number of steps (needed: each step ends in a collective)."""
    idx = list(range(rank, n_items, world))
    per_rank = n_items // world if drop_last else -(-n_items // world)
    if drop_last:
        return idx[:per_rank]
    i = 0
    while len(idx) < per_rank:
        idx.append((rank + i * world) % n_items)
        i += 1
    return idx


def allreduce_sum_(flat: torch.Tensor) -> int:
    """In-place SUM all-reduce of the flat gradient buffer; returns the world size."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        return dist.get_world_size()
    return 1
