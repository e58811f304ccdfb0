"""Convergence check of hybrid parallelism (the reference's tests/convergence/run_hybrid_parallel.py, without wandb /
datasets): a small Bloom is trained on a synthetic, learnable task (noisy counting sequences) with
TensorParallel x DataParallel + ZeRO-1, and every step's loss is printed next to the loss of an identical
single-process model trained on the same global batch.

    torchrun --standalone --nnodes=1 --nproc-per-node 4 examples/convergence_hybrid.py --tp 2 --dp 2 --steps 60
    (CPU: add --backend gloo; GPUs: --backend nccl uses the sm_90a kernels in bf16)
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))  # run from a source checkout

import torch
import torch.distributed as dist

from pipegoose_b200.distributed import ParallelContext, ParallelMode
from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.nn import DataParallel, TensorParallel
from pipegoose_b200.optim import DistributedOptimizer, FusedAdam


def make_batch(step: int, batch: int, seq: int, vocab: int) -> torch.Tensor:
    """Counting sequences ``start, start+3, start+6, ... (mod vocab)`` with 5 % of the positions replaced by noise:
    the next token is a fixed function of the current one, so the loss falls from ln(vocab) towards the noise floor."""
    g = torch.Generator().manual_seed(1000 + step)
    start = torch.randint(0, vocab, (batch, 1), generator=g)
    ids = (start + 3 * torch.arange(seq)[None, :]) % vocab
    noise = torch.rand(batch, seq, generator=g) < 0.05
    return torch.where(noise, torch.randint(0, vocab, (batch, seq), generator=g), ids)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tp", type=int, default=2)
    ap.add_argument("--dp", type=int, default=2)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--batch", type=int, default=16, help="global batch (sequences)")
    ap.add_argument("--seq", type=int, default=64)
    ap.add_argument("--lr", type=float, default=3e-3)
    ap.add_argument("--backend", default="nccl" if torch.cuda.is_available() else "gloo")
    args = ap.parse_args()

    ctx = ParallelContext.from_torch(tensor_parallel_size=args.tp, pipeline_parallel_size=1, data_parallel_size=args.dp,
                                     backend=args.backend)
    rank = ctx.get_global_rank()
    cfg = BloomConfig(vocab_size=256, hidden_size=128, n_layer=2, n_head=4)
    torch.manual_seed(0)
    model = BloomForCausalLM(cfg)
    reference = BloomForCausalLM(cfg)
    reference.load_state_dict(model.state_dict())
    gpu = args.backend == "nccl"
    if gpu:
        model, reference = model.to(torch.bfloat16), reference.to(torch.bfloat16).cuda()
    model = TensorParallel(model, ctx).parallelize()
    model = DataParallel(model, ctx).parallelize()
    if gpu:
        model.to("cuda")
    optim = DistributedOptimizer(FusedAdam(model.parameters(), lr=args.lr), ctx)
    ref_optim = FusedAdam(reference.parameters(), lr=args.lr)
    dev = next(reference.parameters()).device
    dp_rank = ctx.get_local_rank(ParallelMode.DATA)

    first = last = None
    for step in range(args.steps):
        ids = make_batch(step, args.batch, args.seq, cfg.vocab_size).to(dev)
        local = ids.chunk(args.dp)[dp_rank]
        loss = model(local, labels=local).loss
        optim.zero_grad()
        loss.backward()
        optim.step()
        mean = loss.detach().float().clone()
        dist.all_reduce(mean)
        mean = mean.item() / ctx.get_world_size(ParallelMode.GLOBAL)

        ref_loss = reference(ids, labels=ids).loss
        ref_optim.zero_grad()
        ref_loss.backward()
        ref_optim.step()
        if rank == 0 and (step % 5 == 0 or step == args.steps - 1):
            print(f"step {step:3d}  parallel {mean:.4f}  single-process {ref_loss.item():.4f}", flush=True)
        first = mean if first is None else first
        last = mean
    if rank == 0:
        ok = last < 0.6 * first and abs(last - ref_loss.item()) < 0.15 * max(ref_loss.item(), 0.1) + 0.05
        print(f"loss {first:.3f} -> {last:.3f} (single-process {ref_loss.item():.3f}): {'CONVERGED' if ok else 'CHECK'}", flush=True)
    ctx.destroy()


if __name__ == "__main__":
    main()
