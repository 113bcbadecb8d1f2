"""Communication of the K-FAC hot path over torch.distributed (NCCL on the
GPU, gloo in the CPU tests).

Replaces kfac/distributed.py:124-385 (`TorchDistributedCommunicator`): instead
of one async collective per tensor plus flatten/unflatten bucket copies, the
factors / second-order data / preconditioned gradients of all layers live in
contiguous arenas, so each phase is ONE collective per (source, group):

  C1  factor all-reduce (average over the world)     distributed.py:190-246,305-374
  C2  eigenbasis / inverse broadcast in the gradient-worker group   :248-303
  C3  preconditioned-gradient broadcast in the gradient-receiver group

This module is pure plumbing on flat tensors (it works on CPU tensors with
gloo, which is how the world_size-2 tests exercise it); it does no arithmetic
beyond the 1/world averaging of the reference (distributed.py:239-241,369).
"""
from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist


def get_rank(group: Any = None) -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group)
    return 0


def get_world_size(group: Any = None) -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group)
    return 1


class NonSquareTensorError(Exception):
    """Raised when a non-square tensor is passed to a symmetric operation."""


class ArenaCommunicator:
    """Collectives on flat arena slices.

    `bucket_cap_mb` is kept for API compatibility with the reference
    constructor (preconditioner.py:232); the arena already is the bucket, so
    it only bounds the size of a single collective call when > 0.
    """

    def __init__(self, bucket_cap_mb: float = 25.0) -> None:
        if bucket_cap_mb < 0:
            raise ValueError('bucket_cap_mb must be >= 0')
        self.bucket_cap_mb = bucket_cap_mb
        self.calls = {'allreduce': 0, 'broadcast': 0}

    def allreduce_average(self, flat: torch.Tensor, group: Any = None) -> None:
        """In-place sum over `group` then multiply by 1/size; no-op at size 1
        (kfac/distributed.py:221-222)."""
        size = get_world_size(group)
        if size == 1:
            return
        assert flat.is_contiguous()
        self.calls['allreduce'] += 1
        backend = dist.get_backend(group)
        if backend == 'nccl':
            dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=group)
        else:
            dist.all_reduce(flat, group=group)
            flat.mul_(1.0 / size)

    def broadcast(self, flat: torch.Tensor, src: int, group: Any = None) -> None:
        """In-place broadcast from global rank `src`; no-op at size 1
        (kfac/distributed.py:275-277)."""
        if get_world_size(group) == 1:
            return
        assert flat.is_contiguous()
        self.calls['broadcast'] += 1
        dist.broadcast(flat, src=src, group=group)

    def fence(self, token: torch.Tensor, group: Any = None) -> None:
        """Group-wide ordering point after peer-to-peer stores: a one-element all-reduce (its
        kernel starts after this rank's prior work on the stream and completes only when every
        rank of the group has reached it)."""
        if get_world_size(group) == 1:
            return
        self.calls['fence'] = self.calls.get('fence', 0) + 1
        dist.all_reduce(token, group=group)

    # reference-compatible no-op (the arena design has no pending buckets)
    def flush_allreduce_buckets(self) -> None:
        return None


def triu_numel(n: int) -> int:
    return n * (n + 1) // 2
