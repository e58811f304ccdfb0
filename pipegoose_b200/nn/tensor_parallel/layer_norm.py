"""LayerNorm under tensor parallelism (parity: reference nn/tensor_parallel/layer_norm.py:8-25): parameters are
replicated, nothing is communicated.  It is ``torch.nn.LayerNorm`` plus a fast path — CUDA bf16 rows go through the fused
sm_90a LayerNorm kernel (ops/kernels.py) — which also makes the class swap of ``TensorParallel`` a plain
subclass swap that ``deparallelize()`` can undo."""
from __future__ import annotations

import torch
from torch import nn

from pipegoose_b200.distributed.parallel_context import ParallelContext


class LayerNorm(nn.LayerNorm):
    def __init__(self, normalized_shape, eps: float = 1e-5, bias: bool = True, parallel_context: ParallelContext = None):
        super().__init__(normalized_shape, eps=eps, elementwise_affine=True, bias=bias)
        self.parallel_context = parallel_context

    def _kernel_eligible(self, x: torch.Tensor) -> bool:
        return (x.is_cuda and x.dtype == torch.bfloat16 and self.bias is not None and len(self.normalized_shape) == 1
                and x.shape[-1] % 8 == 0)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        if self._kernel_eligible(input):
            from pipegoose_b200.models.bloom import fused_layer_norm

            return fused_layer_norm(input, self.weight, self.bias, self.eps)
        return nn.LayerNorm.forward(self, input)
