"""DiLoCo: data-parallel replicas that only talk every H steps (pipegoose_b200.optim.DiLoCoOptimizer) — the regime the
reference's README names as its goal.  Each worker (a DATA-group rank, tensor-parallel inside if --tp > 1) trains on its
own synthetic shard with its own FusedAdam; every --inner-steps steps the workers average their displacement and an outer
Nesterov SGD moves the shared parameters.

    torchrun --standalone --nnodes=1 --nproc-per-node 4 examples/diloco.py --tp 2 --workers 2 --backend gloo   # CPU
    torchrun --standalone --nnodes=1 --nproc-per-node 8 examples/diloco.py --tp 2 --workers 4                  # H100s
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))  # run from a source checkout

import torch
import torch.distributed as dist

from pipegoose_b200.distributed import ParallelContext, ParallelMode
from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.nn import TensorParallel
from pipegoose_b200.optim import DiLoCoOptimizer, FusedAdam


def batch_for(worker: int, step: int, batch: int, seq: int, vocab: int) -> torch.Tensor:
    """Counting sequences (next token = current + 3 mod vocab) — every worker sees different starts."""
    g = torch.Generator().manual_seed(10_000 * worker + step)
    start = torch.randint(0, vocab, (batch, 1), generator=g)
    return (start + 3 * torch.arange(seq)[None, :]) % vocab


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tp", type=int, default=1)
    ap.add_argument("--workers", type=int, default=2)
    ap.add_argument("--inner-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--backend", default="nccl" if torch.cuda.is_available() else "gloo")
    args = ap.parse_args()

    ctx = ParallelContext.from_torch(tensor_parallel_size=args.tp, pipeline_parallel_size=1, data_parallel_size=args.workers,
                                     backend=args.backend)
    cfg = BloomConfig(vocab_size=256, hidden_size=128, n_layer=2, n_head=4)
    torch.manual_seed(0)
    model = BloomForCausalLM(cfg)
    gpu = args.backend == "nccl"
    if gpu:
        model = model.to(torch.bfloat16)
    model = TensorParallel(model, ctx).parallelize()   # NOT DataParallel: the workers do not share gradients
    if gpu:
        model.to("cuda")
    optim = DiLoCoOptimizer(FusedAdam(model.parameters(), lr=3e-3), ctx, inner_steps=args.inner_steps, outer_lr=0.7,
                            outer_momentum=0.9)
    worker = ctx.get_local_rank(ParallelMode.DATA)
    dev = next(model.parameters()).device
    for step in range(args.rounds * args.inner_steps):
        ids = batch_for(worker, step, 8, 32, cfg.vocab_size).to(dev)
        loss = model(ids, labels=ids).loss
        optim.zero_grad()
        loss.backward()
        optim.step()
        if (step + 1) % args.inner_steps == 0:
            mean = loss.detach().float().clone()
            dist.all_reduce(mean)
            if ctx.get_global_rank() == 0:
                print(f"outer step {optim.outer_step_count:2d} (after {step + 1:3d} local steps, "
                      f"{optim.outer_step_count} parameter exchanges)  mean worker loss {mean.item() / dist.get_world_size():.4f}",
                      flush=True)
    ctx.destroy()


if __name__ == "__main__":
    main()
