"""Switch-style mixture of experts on Bloom: experts sharded over the tensor group.

    torchrun --standalone --nnodes=1 --nproc-per-node 2 examples/moe.py --tp 2 --experts 4
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))  # run from a source checkout

import torch

from pipegoose_b200.distributed import ParallelContext
from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.nn import DataParallel, ExpertParallel, TensorParallel
from pipegoose_b200.nn.expert_parallel import ExpertContext, SwitchNoisePolicy, Top1Router
from pipegoose_b200.optim import DistributedOptimizer, FusedAdam

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--tp", type=int, default=2)
    ap.add_argument("--dp", type=int, default=1)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--backend", default="gloo")
    args = ap.parse_args()
    ctx = ParallelContext.from_torch(tensor_parallel_size=args.tp, pipeline_parallel_size=1, data_parallel_size=args.dp,
                                     backend=args.backend)
    cfg = BloomConfig(vocab_size=1024, hidden_size=128, n_layer=4, n_head=8)
    model = BloomForCausalLM(cfg)
    router = Top1Router(SwitchNoisePolicy(), args.experts, cfg.hidden_size, expert_capacity=(1.25, 2.0))
    gpu = args.backend == "nccl"
    if gpu:  # bf16 on the GPU path: router kernel + NVLink dispatch + grouped wgmma expert GEMMs
        model, router = model.to(torch.bfloat16), router.to(torch.bfloat16)
    model = ExpertParallel(model, args.experts, mapping=[0, 2], router=router, parallel_context=ctx).parallelize()
    model = TensorParallel(model, ctx).parallelize()
    model = DataParallel(model, ctx).parallelize()
    if gpu:
        model.to("cuda")
    optim = DistributedOptimizer(FusedAdam(model.parameters(), lr=3e-3), ctx) if gpu \
        else torch.optim.Adam(model.parameters(), lr=3e-3)
    expert_ctx = ExpertContext.get_instance()

    def make_batch(step, batch=8, seq=32):
        """Noisy counting sequences (learnable): next token = current + 3 (mod vocab), 5 % noise."""
        g = torch.Generator().manual_seed(1000 + step)
        start = torch.randint(0, cfg.vocab_size, (batch, 1), generator=g)
        ids = (start + 3 * torch.arange(seq)[None, :]) % cfg.vocab_size
        noise = torch.rand(batch, seq, generator=g) < 0.05
        return torch.where(noise, torch.randint(0, cfg.vocab_size, (batch, seq), generator=g), ids)

    for step in range(args.steps):
        ids = make_batch(step)
        if gpu:
            ids = ids.cuda()
        loss = model(ids, labels=ids).loss
        loss = loss + 0.01 * sum(expert_ctx.pop_all_aux_loss()) + 0.001 * sum(expert_ctx.pop_all_z_loss())
        optim.zero_grad()
        loss.backward()
        optim.step()
        if ctx.get_global_rank() == 0 and (step % 5 == 0 or step == args.steps - 1):
            print(f"step {step} loss {loss.item():.4f}", flush=True)
    ctx.destroy()
