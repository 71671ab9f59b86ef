"""Data-parallel plumbing (one process per GPU, torch.distributed over NCCL/NVLink; gloo on CPU in tests).

The path shards by batch (SURVEY 8(e)): every sample is independent (GroupNorm, attention are per sample), so the only
exchange is ONE sum all-reduce of the flat fp32 gradient bucket between backward and Adam; 1/world is folded into the
Adam kernel.  The reference's pmap step has no collective at all (train.py:49-76)."""
from __future__ import annotations

import os
from typing import Dict

import torch
import torch.distributed as dist


def is_dist() -> bool:
    return dist.is_available() and dist.is_initialized()


def world_size() -> int:
    return dist.get_world_size() if is_dist() else 1


def rank() -> int:
    return dist.get_rank() if is_dist() else 0


def init_from_env(backend: str = 'nccl') -> int:
    """torchrun-style initialisation (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*).  Returns the local rank."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not is_dist():
        if backend == 'nccl':
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device('cuda', local))
        else:
            dist.init_process_group(backend)
    elif backend == 'nccl' and torch.cuda.is_available():
        torch.cuda.set_device(local)
    return local


def shard_batch(batch: Dict[str, object], r: int, world: int) -> Dict[str, object]:
    """Splits the leading (batch) axis of every array evenly: rank r gets rows [r*B/world, (r+1)*B/world)."""
    out = {}
    for k, v in batch.items():
        n = len(v)
        if n % world != 0:
            raise ValueError(f"batch['{k}'] of size {n} does not split over {world} ranks")
        per = n // world
        out[k] = v[r * per:(r + 1) * per]
    return out


def broadcast_params(flat: torch.Tensor, src: int = 0) -> None:
    if world_size() > 1:
        dist.broadcast(flat, src=src)


def allreduce_sum_(flat: torch.Tensor, bucket_elems: int = 0) -> None:
    """Sum all-reduce of the flat gradient buffer, optionally in buckets (async, then waited) so large models overlap
    NVLink transfers of one bucket with the reduction of the next."""
    if world_size() == 1:
        return
    if bucket_elems <= 0 or bucket_elems >= flat.numel():
        dist.all_reduce(flat)
        return
    works = [dist.all_reduce(flat[i:i + bucket_elems], async_op=True) for i in range(0, flat.numel(), bucket_elems)]
    for w in works:
        w.wait()


class GradReducer:
    """Bucketed sum all-reduce of the flat gradient buffer, driven by the backward's bucket hook.

    The engine calls `on_bucket(offset, n)` (Engine.set_bucket_callback) as soon as grads[offset:offset+n] is final, while
    the rest of the backward is still being enqueued; each bucket is reduced asynchronously on the process group's
    communication stream (NCCL over NVLink), ordered after the compute stream's current point, so the transfer of the
    up-path gradients overlaps the down-path backward.  `wait()` orders the compute stream after all of them (no host
    block on NCCL).  Under CUDA-graph capture both calls are captured with the step."""

    def __init__(self, flat_grads: torch.Tensor, group=None):
        self.flat = flat_grads
        self.group = group
        self.works = []
        self.enabled = True
        self.ranges = []          # (offset, n) of the last backward, for reporting

    def begin(self) -> None:
        self.works, self.ranges = [], []

    def on_bucket(self, offset: int, n: int) -> None:
        self.ranges.append((offset, n))
        if not self.enabled or world_size() == 1:
            return
        self.works.append(dist.all_reduce(self.flat[offset:offset + n], group=self.group, async_op=True))

    def wait(self) -> None:
        for w in self.works:
            w.wait()
        self.works = []


def max_over_ranks(value: float) -> float:
    if world_size() == 1:
        return float(value)
    dev = 'cuda' if dist.get_backend() == 'nccl' else 'cpu'
    t = torch.tensor([float(value)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def all_gather_object(obj) -> list:
    """Every rank's picklable `obj`, indexed by rank (gloo and NCCL)."""
    if world_size() == 1:
        return [obj]
    out = [None] * world_size()
    dist.all_gather_object(out, obj)
    return out


def barrier() -> None:
    if world_size() > 1:
        dist.barrier()
