"""Sequence-parallel tensor-parallel communicator used by the fused sub-layer functions.

Library mode (``fused=False``): NCCL/gloo all-gather / reduce-scatter around plain GEMMs — the
correctness baseline, and what CPU tests run.  Fused mode (``fused=True``): the hand-written
sm_90a kernels in which the collective is part of the GEMM (``pipegoose_b200.ops.comm``):

    ag_gemm     all-gather -> GEMM      (column-parallel forward, row-parallel dgrad)
    gemm_rs     GEMM -> reduce-scatter  (row-parallel forward, column-parallel dgrad)
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from pipegoose_b200.distributed.parallel_mode import ParallelMode


class TensorParallelComm:
    def __init__(self, parallel_context, parallel_mode: ParallelMode = ParallelMode.TENSOR, fused=None):
        self.ctx = parallel_context
        self.mode = parallel_mode
        self.group = parallel_context.get_group(parallel_mode)
        self.size = parallel_context.get_world_size(parallel_mode)
        self.rank = parallel_context.get_local_rank(parallel_mode)
        self._engine = None
        want = os.environ.get("PIPEGOOSE_B200_FUSED_TP", "1") == "1" if fused is None else fused
        self.fused = False
        self._want_fused = want and dist.get_backend(self.group) == "nccl" and torch.cuda.is_available()

    def enable_fused(self):
        """Create the NVLink peer-memory engine (symmetric workspace + fused kernels); collective call."""
        if self._want_fused and self._engine is None:
            from pipegoose_b200.distributed.symmetric import peers_share_a_node
            from pipegoose_b200.ops.comm import FusedTPEngine

            if not peers_share_a_node(self.ctx, self.mode):   # a tensor group across hosts: NCCL collectives + plain GEMMs
                self._want_fused = False
                return

            self._engine = FusedTPEngine(self)
            self.fused = True

    # 1: the collectives that have no GEMM to be fused into (vocab-parallel embedding reduce-scatter / all-gather, the
    # cross-entropy statistics exchange, the partial-gradient sum) run on the NVLink peer-memory kernels as well, so a
    # tensor-parallel step contains no NCCL kernel.  Covered by tests/test_gpu_multi.py::test_tp2_bloom* (2 GPUs).
    PEER_COLLECTIVES = os.environ.get("PIPEGOOSE_B200_TP_PEER_COLLECTIVES", "1") == "1"

    def _peer_ok(self, x: torch.Tensor) -> bool:
        return (self.fused and self.PEER_COLLECTIVES and x.is_cuda and x.dtype in (torch.bfloat16, torch.float32)
                and x.dim() >= 1 and (x.numel() * x.element_size()) % 16 == 0 and x.numel() > 0)

    # ------------------------------------------------------------------ library collectives
    def all_gather_rows(self, x: torch.Tensor) -> torch.Tensor:
        x = x.detach().contiguous()
        if self._peer_ok(x):
            # (a copy: the engine's gathered buffer is recycled two calls later, the caller may keep the result)
            return self._engine.all_gather_rows(x).clone()
        out = torch.empty((x.shape[0] * self.size,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x, group=self.group)
        return out

    def all_gather_stack(self, x: torch.Tensor) -> torch.Tensor:
        return self.all_gather_rows(x.unsqueeze(0))

    def all_gather_cols(self, x: torch.Tensor) -> torch.Tensor:
        full = self.all_gather_rows(x.unsqueeze(0))  # [T, M, n]
        return full.permute(1, 0, 2).reshape(x.shape[0], -1)

    def reduce_scatter_rows(self, x: torch.Tensor) -> torch.Tensor:
        x = x.detach().contiguous()
        assert x.shape[0] % self.size == 0
        rows = x.shape[0] // self.size
        if self._peer_ok(x) and x.dtype == torch.bfloat16 and x.dim() == 2 and (rows * x.shape[1]) % 8 == 0:
            return self._engine.reduce_scatter_rows(x)
        if dist.get_backend(self.group) == "gloo":
            dist.all_reduce(x, group=self.group)
            return x[self.rank * rows:(self.rank + 1) * rows].clone()
        out = torch.empty((rows,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.reduce_scatter_tensor(out, x, group=self.group)
        return out

    def all_reduce(self, x: torch.Tensor) -> torch.Tensor:
        if self._peer_ok(x) and x.dtype == torch.float32 and x.is_contiguous() and x.numel() <= (1 << 24):
            return self._engine.all_reduce_f32_(x)
        dist.all_reduce(x, group=self.group)
        return x

    # differentiable forms (used outside the fused sub-layer functions, e.g. the logits path)
    def gather_rows(self, x: torch.Tensor) -> torch.Tensor:
        return _GatherRows.apply(x, self)

    def gather_cols(self, x: torch.Tensor) -> torch.Tensor:
        return _GatherCols.apply(x, self)

    def scatter_rows(self, x: torch.Tensor) -> torch.Tensor:
        """Sum partial ``[tokens, h]`` results over the group and keep this rank's token block (the conjugate of
        :meth:`gather_rows`: reduce-scatter forward, all-gather backward)."""
        return _ScatterRows.apply(x, self)

    # ------------------------------------------------------------------ fused kernels
    def ag_input_buffer(self, rows_local: int, cols: int):
        return self._engine.ag_input_buffer(rows_local, cols) if self.fused else None

    def ag_gemm(self, x_shard, weight, bias=None, gelu=False, aux_holder=None, extra=None):
        return self._engine.ag_gemm(x_shard, weight, bias, gelu, aux_holder, extra=extra)

    def gemm_rs(self, a, weight, bias=None, residual=None):
        return self._engine.gemm_rs(a, weight, bias, residual)

    def ag_gemm_nn(self, dy_shard, weight, dgelu_aux=None):
        return self._engine.ag_gemm_nn(dy_shard, weight, dgelu_aux)

    def gemm_rs_nn(self, dy, weight):
        return self._engine.gemm_rs_nn(dy, weight)


class _GatherRows(torch.autograd.Function):
    """all-gather along tokens; backward reduce-scatters the gradient."""

    @staticmethod
    def forward(ctx, x, comm):
        ctx.comm = comm
        return comm.all_gather_rows(x)

    @staticmethod
    def backward(ctx, g):
        return ctx.comm.reduce_scatter_rows(g), None


class _ScatterRows(torch.autograd.Function):
    """reduce-scatter along tokens; backward all-gathers the gradient."""

    @staticmethod
    def forward(ctx, x, comm):
        ctx.comm = comm
        return comm.reduce_scatter_rows(x.contiguous())

    @staticmethod
    def backward(ctx, g):
        return ctx.comm.all_gather_rows(g.contiguous()), None


class _GatherCols(torch.autograd.Function):
    """all-gather along features (every rank uses the full result); backward keeps the local slice."""

    @staticmethod
    def forward(ctx, x, comm):
        ctx.comm, ctx.width = comm, x.shape[-1]
        return comm.all_gather_cols(x)

    @staticmethod
    def backward(ctx, g):
        r = ctx.comm.rank
        return g[:, r * ctx.width:(r + 1) * ctx.width].contiguous(), None
