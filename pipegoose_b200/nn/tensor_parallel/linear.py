"""1-D (Megatron-style) tensor-parallel linear layers with the reference's replicated-activation contract (parity:
reference nn/tensor_parallel/linear.py:17-82): a column-parallel layer owns a block of output features (optionally
all-gathers them), a row-parallel layer owns a block of input features and all-reduces its partial products.

Both are one class body: what differs is the weight dimension that is split (``shard_dim``) and the pair of
communication ops around the local GEMM, which runs on the wgmma kernel with the bias in its epilogue
(``ops.functional.linear``).  The sequence-parallel fast path with fused all-gather→GEMM / GEMM→reduce-scatter kernels
lives in ``pipegoose_b200.models`` / ``ops/functional.py``; these layers exist so that any 🤗 model can be sharded.
"""
from __future__ import annotations

import torch
from torch import nn

from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.nn.tensor_parallel import _functional as comm
from pipegoose_b200.ops.functional import linear as fused_linear


class _ShardedLinear(nn.Module):
    shard_dim = 0  # dimension of the [out, in] weight that is split over the tensor group

    def __init__(self, in_features: int, out_features: int, bias: bool, parallel_context: ParallelContext):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.parallel_context = parallel_context
        group = parallel_context.get_world_size(ParallelMode.TENSOR) if parallel_context is not None else 1
        shape = [out_features, in_features]
        what = ("out_features", "in_features")[self.shard_dim]
        assert shape[self.shard_dim] % group == 0, f"{what} must be divisible by the tensor parallel size"
        shape[self.shard_dim] //= group
        self.weight = nn.Parameter(torch.empty(shape))
        nn.init.normal_(self.weight, std=0.02)
        self.bias = nn.Parameter(torch.zeros(shape[0])) if bias else None  # row-parallel: the full-width bias

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, local_weight={tuple(self.weight.shape)}"


class ColumnParallelLinear(_ShardedLinear):
    shard_dim = 0

    def __init__(self, in_features: int, out_features: int, bias: bool = True, gather_output: bool = False,
                 parallel_context: ParallelContext = None):
        super().__init__(in_features, out_features, bias, parallel_context)
        self.gather_output = gather_output

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        replicated = comm.broadcast_to_tensor_group(input, self.parallel_context)       # identity fwd / all-reduce bwd
        local = fused_linear(replicated, self.weight, self.bias)
        if not self.gather_output:
            return local
        full = comm.gather_to_tensor_group(local, dim=-1, parallel_context=self.parallel_context)
        keep = getattr(self, "unpadded_out_features", None)   # an LM head whose vocabulary was padded to split evenly
        return full if keep is None or keep == full.shape[-1] else full[..., :keep]


class RowParallelLinear(_ShardedLinear):
    shard_dim = 1

    def __init__(self, in_features: int, out_features: int, bias: bool = True, parallel_context: ParallelContext = None):
        super().__init__(in_features, out_features, bias, parallel_context)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        mine = comm.scatter_to_tensor_group(input, dim=-1, parallel_context=self.parallel_context)
        total = comm.reduce_to_tensor_group(fused_linear(mine, self.weight, None), self.parallel_context)
        return total if self.bias is None else total + self.bias  # bias once, after the sum
