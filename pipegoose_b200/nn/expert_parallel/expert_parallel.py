"""``ExpertParallel`` wrapper (parity: reference nn/expert_parallel/expert_parallel.py:13-83):
turn the MLPs of selected transformer blocks into mixture-of-experts layers whose experts are
sharded over the TENSOR group."""
from __future__ import annotations

import os
import re
from typing import List, Optional

import torch
from torch import nn

from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer
from pipegoose_b200.nn.parallel import Parallel


class ExpertParallel(Parallel):
    def __init__(self, module: nn.Module, num_experts: int, expert: Optional[nn.Module] = None,
                 mapping: Optional[List[int]] = None, router: nn.Module = None,
                 enable_tensor_parallelism: bool = False, parallel_context: ParallelContext = None,
                 fused: Optional[bool] = None):
        super().__init__(module, parallel_context)
        tensor_parallel_size = parallel_context.get_world_size(ParallelMode.TENSOR)
        assert num_experts % tensor_parallel_size == 0, \
            "the number of experts must be divisible by the tensor parallel size"
        num_layers = self._num_blocks(module)
        if mapping is None:  # reference Q6: default to every layer (applied before validating)
            mapping = list(range(num_layers))
        assert all(0 <= i < num_layers for i in mapping), "a mapped layer index does not exist in the model"
        assert router is not None, "a router is required"
        self.num_experts = num_experts
        self.expert = expert
        self.mapping = mapping
        self.router = router
        self.enable_tensor_parallelism = enable_tensor_parallelism
        self.fused = fused

    # where the transformer blocks live: Bloom / GPT-2 (the reference's only case, expert_parallel.py:60-66), LLaMA-style
    # decoders and GPT-NeoX; a block qualifies when it has an ``mlp`` child to replace
    BLOCK_PATTERN = re.compile(r"^(?:transformer\.h|model\.layers|gpt_neox\.layers)\.(\d+)$")

    @classmethod
    def _blocks(cls, module: nn.Module):
        return [(int(cls.BLOCK_PATTERN.match(n).group(1)), m) for n, m in module.named_modules()
                if cls.BLOCK_PATTERN.match(n) and hasattr(m, "mlp")]

    @classmethod
    def _num_blocks(cls, module: nn.Module) -> int:
        return len(cls._blocks(module))

    @torch.no_grad()
    def parallelize(self) -> nn.Module:
        for layer_idx, block in self._blocks(self.module):
            if layer_idx not in self.mapping:
                continue
            expert = self.expert if self.expert is not None else block.mlp
            if self._use_fused(expert):
                # NVLink all-to-all dispatch/combine + grouped wgmma expert GEMMs (ops/moe.py)
                from pipegoose_b200.ops.moe import FusedExpertLayer

                block.mlp = FusedExpertLayer(self.num_experts, expert, self.router, self.parallel_context)
            else:
                block.mlp = ExpertLayer(self.num_experts, expert, self.router, self.enable_tensor_parallelism,
                                        self.parallel_context)
        return self.module

    def _use_fused(self, expert: nn.Module) -> bool:
        """Fused path: pipegoose_b200 Bloom (token-sharded 2-D activations), BloomMLP experts, a Top-k
        router with a linear gate, NCCL/CUDA.  ``fused=None`` picks it automatically."""
        import torch.distributed as dist

        from pipegoose_b200.models.bloom import BloomMLP

        if self.fused is False or self.enable_tensor_parallelism:
            return False
        if self.fused is None and os.environ.get("PIPEGOOSE_B200_FUSED_MOE", "1") == "0":
            # the switch bench.py's numerics self-check flips next to PIPEGOOSE_B200_FUSED_TP / _FUSED_DP: ExpertLayer
            # (library collectives around plain kernels) instead of the fused NVLink dispatch / combine layer
            return False
        ok = (isinstance(expert, BloomMLP) and hasattr(self.module, "hidden_states") and hasattr(self.router, "gate")
              and torch.cuda.is_available()
              and dist.get_backend(self.parallel_context.get_group(ParallelMode.TENSOR)) == "nccl")
        if ok:
            from pipegoose_b200.distributed.symmetric import peers_share_a_node

            ok = peers_share_a_node(self.parallel_context, ParallelMode.TENSOR)   # NVLink all-to-all needs one host
        if self.fused is True and not ok:
            raise ValueError("fused=True needs a pipegoose_b200 Bloom model, BloomMLP experts, a gate router and NCCL")
        return ok

    @torch.no_grad()
    def deparallelize(self) -> nn.Module:
        """Undo the expert *sharding* (unimplemented in the reference): afterwards every rank holds all the experts
        of every MoE layer and runs them locally — the layers stay mixture-of-experts layers (a trained MoE cannot
        be folded back into one dense MLP), but the module no longer needs the TENSOR group, e.g. to export one
        consolidated checkpoint.  Fused layers are converted to plain ``ExpertLayer``s first."""
        for _, block in self._blocks(self.module):
            mlp = getattr(block, "mlp", None)
            if isinstance(mlp, ExpertLayer):
                mlp.gather_experts_()
            elif hasattr(mlp, "to_expert_layer"):
                block.mlp = mlp.to_expert_layer().gather_experts_()
        return self.module
