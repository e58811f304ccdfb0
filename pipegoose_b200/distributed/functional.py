"""Collectives keyed by ``(parallel_context, parallel_mode)`` (parity: reference
distributed/functional.py:30-182).  Every function is a no-op for a group of one.

These are the *library* collectives (NCCL / gloo through torch.distributed): they are the
plumbing and the always-correct fallback.  The hot paths of the parallel wrappers use the fused
sm_90a kernels in ``pipegoose_b200.ops`` instead and only fall back to these on CPU/gloo.
``reduce_scatter`` and ``all_to_all`` exist here (the reference left the former as a stub and has
no all-to-all at all).
"""
from __future__ import annotations

from typing import Any, Optional

import torch
import torch.distributed as dist
from torch.distributed import ReduceOp

from pipegoose_b200.distributed._p2p import _P2P
from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode


def _maybe_async(result, work, async_op):
    return (result, work) if async_op else result


def scatter(tensor: torch.Tensor, dim: int, parallel_context: Optional[ParallelContext] = None,
            parallel_mode: Optional[ParallelMode] = None) -> torch.Tensor:
    """Keep this rank's slice of ``tensor`` along ``dim`` (no communication)."""
    world_size = parallel_context.get_world_size(parallel_mode)
    if world_size == 1:
        return tensor
    assert tensor.size(dim) % world_size == 0, "the scattered dimension must divide evenly"
    rank = parallel_context.get_local_rank(parallel_mode)
    width = tensor.size(dim) // world_size
    return tensor.narrow(dim, rank * width, width)


def reduce(tensor: torch.Tensor, dst: int, op: ReduceOp = ReduceOp.SUM, async_op: bool = False,
           parallel_context: Optional[ParallelContext] = None, parallel_mode: Optional[ParallelMode] = None):
    """Reduce onto ``dst`` — a GLOBAL rank that belongs to the group, as in ``torch.distributed`` and in the reference
    (functional.py:49-69; its tests pass ``get_ranks_in_group(mode)[-1]``)."""
    if parallel_context.get_world_size(parallel_mode) == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    assert dst in parallel_context.get_ranks_in_group(parallel_mode), f"global rank {dst} is not in this {parallel_mode} group"
    work = dist.reduce(tensor, dst=dst, op=op, group=group, async_op=async_op)
    return _maybe_async(tensor, work, async_op)


def broadcast(tensor: torch.Tensor, src: int, async_op: bool = False,
              parallel_context: Optional[ParallelContext] = None, parallel_mode: Optional[ParallelMode] = None):
    """Broadcast from ``src`` — a GLOBAL rank that belongs to the group (reference functional.py:72-91)."""
    if parallel_context.get_world_size(parallel_mode) == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    assert src in parallel_context.get_ranks_in_group(parallel_mode), f"global rank {src} is not in this {parallel_mode} group"
    work = dist.broadcast(tensor, src=src, group=group, async_op=async_op)
    return _maybe_async(tensor, work, async_op)


def all_gather(tensor: torch.Tensor, dim: int = 0, async_op: bool = False,
               parallel_context: Optional[ParallelContext] = None, parallel_mode: Optional[ParallelMode] = None):
    """Concatenate every rank's ``tensor`` along ``dim``.

    Gathers straight into one output buffer (``all_gather_into_tensor``) and only permutes when
    ``dim`` is not the leading one; the reference gathers into a python list and ``torch.cat``s.
    """
    world_size = parallel_context.get_world_size(parallel_mode)
    if world_size == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    src = tensor.detach()    # (the collective is not differentiable; a tensor that requires grad must not reach gloo's
    src = src.unsqueeze(0) if src.dim() == 0 else src   # in-place chunk copies — reference tests pass such tensors)
    src = src.contiguous()
    d = dim % src.dim()
    flat2d = torch.empty((world_size * src.shape[0],) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    work = dist.all_gather_into_tensor(flat2d, src, group=group, async_op=async_op)
    flat = flat2d.view((world_size,) + tuple(src.shape))

    def finish():
        if d == 0:
            return flat.reshape((world_size * src.shape[0],) + tuple(src.shape[1:]))
        out = flat.movedim(0, d)  # [..., world, src.shape[d], ...]
        shape = list(src.shape)
        shape[d] *= world_size
        return out.reshape(shape)

    if async_op:
        if d == 0:
            return finish(), work   # a view of the gather buffer: valid once ``work.wait()`` returned
        # the permute to ``dim`` COPIES the gather buffer, so it may only run after the collective completed: the
        # result is gathered along dim 0 into ``out`` now and put in place by ``wait()``
        shape = list(src.shape)
        shape[d] *= world_size
        out = torch.empty(shape, dtype=src.dtype, device=src.device)
        return out, _DeferredWork(work, lambda: out.copy_(finish()))
    return finish()


class _DeferredWork:
    """``Work``-like handle whose ``wait()`` first waits for the collective and then runs a post-processing step."""

    def __init__(self, work, after=None):
        self._work, self._after = work, after

    def wait(self, *args, **kwargs):
        if self._work is not None:
            self._work.wait(*args, **kwargs)
            self._work = None
        if self._after is not None:
            after, self._after = self._after, None
            after()
        return True

    def is_completed(self):
        return self._work is None or self._work.is_completed()


def all_reduce(tensor: torch.Tensor, op: ReduceOp = ReduceOp.SUM, async_op: bool = False,
               parallel_context: Optional[ParallelContext] = None, parallel_mode: Optional[ParallelMode] = None):
    if parallel_context.get_world_size(parallel_mode) == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    work = dist.all_reduce(tensor, op=op, group=group, async_op=async_op)
    return _maybe_async(tensor, work, async_op)


def reduce_scatter(tensor: torch.Tensor, dim: int = 0, op: ReduceOp = ReduceOp.SUM, async_op: bool = False,
                   parallel_context: Optional[ParallelContext] = None, parallel_mode: Optional[ParallelMode] = None):
    """Reduce across the group and keep this rank's slice along ``dim``."""
    world_size = parallel_context.get_world_size(parallel_mode)
    if world_size == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    d = dim % tensor.dim()
    assert tensor.size(d) % world_size == 0, "the scattered dimension must divide evenly"
    src = tensor.movedim(d, 0).contiguous() if d != 0 else tensor.contiguous()
    out = torch.empty((src.shape[0] // world_size,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    if dist.get_backend(group) == "gloo":
        # gloo has no reduce_scatter: all-reduce a COPY (the caller's tensor is an input, not scratch) then slice
        if src.data_ptr() == tensor.data_ptr():
            src = src.clone()
        dist.all_reduce(src, op=op, group=group)
        rank = parallel_context.get_local_rank(parallel_mode)
        out.copy_(src.narrow(0, rank * out.shape[0], out.shape[0]))
        work = _DeferredWork(None) if async_op else None   # already complete
    else:
        work = dist.reduce_scatter_tensor(out, src, op=op, group=group, async_op=async_op)
    result = out.movedim(0, d) if d != 0 else out
    return _maybe_async(result, work, async_op)


def all_to_all(tensor: torch.Tensor, parallel_context: Optional[ParallelContext] = None,
               parallel_mode: Optional[ParallelMode] = None, output_split_sizes=None, input_split_sizes=None):
    """Exchange dim-0 slices with every rank of the group (equal or explicit split sizes)."""
    world_size = parallel_context.get_world_size(parallel_mode)
    if world_size == 1:
        return tensor
    group = parallel_context.get_group(parallel_mode)
    tensor = tensor.contiguous()
    if output_split_sizes is None:
        out = torch.empty_like(tensor)
    else:
        out = torch.empty((sum(output_split_sizes),) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    if dist.get_backend(group) == "gloo":
        # gloo lacks all_to_all_single on some builds: emulate with all_gather of padded slices
        rank = parallel_context.get_local_rank(parallel_mode)
        in_sizes = input_split_sizes or [tensor.shape[0] // world_size] * world_size
        out_sizes = output_split_sizes or [tensor.shape[0] // world_size] * world_size
        max_rows = torch.tensor([max(in_sizes)], dtype=torch.long)
        dist.all_reduce(max_rows, op=ReduceOp.MAX, group=group)
        pad = int(max_rows.item())
        send = tensor.new_zeros((world_size, pad) + tuple(tensor.shape[1:]))
        off = 0
        for r, n in enumerate(in_sizes):
            send[r, :n] = tensor[off:off + n]
            off += n
        gathered = [torch.empty_like(send) for _ in range(world_size)]
        dist.all_gather(gathered, send, group=group)
        off = 0
        for r, n in enumerate(out_sizes):
            out[off:off + n] = gathered[r][rank, :n]
            off += n
        return out
    dist.all_to_all_single(out, tensor, output_split_sizes=output_split_sizes,
                           input_split_sizes=input_split_sizes, group=group)
    return out


def send(data: Any, src: int, dst: int, parallel_context: ParallelContext,
         parallel_mode: ParallelMode = ParallelMode.PIPELINE):
    """P2P: the rank whose local rank is ``src`` sends ``data`` to local rank ``dst``."""
    if src == parallel_context.get_local_rank(parallel_mode):
        _P2P().send(data, dst, parallel_context, parallel_mode)


def recv(src: int, dst: int, parallel_context: ParallelContext,
         parallel_mode: ParallelMode = ParallelMode.PIPELINE) -> Optional[Any]:
    """P2P: the rank whose local rank is ``dst`` receives from local rank ``src``."""
    if dst == parallel_context.get_local_rank(parallel_mode):
        return _P2P().recv(src, parallel_context, parallel_mode)
    return None


def barrier(parallel_context: ParallelContext, parallel_mode: ParallelMode):
    dist.barrier(group=parallel_context.get_group(parallel_mode))
