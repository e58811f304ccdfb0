"""Loss curves on GPUs: this library next to the reference on the same learnable synthetic task (the reference's own
"benchmarks" are convergence runs: tests/convergence/run_hybrid_parallel.py, run_ep.py — wandb + imdb, neither
available offline).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29541 \
        tools/convergence_gpu.py --gpus 4 --steps 300                       # TP2 x DP2 + ZeRO-1, fused kernels
    ... tools/convergence_gpu.py --gpus 4 --steps 300 --impl reference      # the reference's stock path, same task
    ... tools/convergence_gpu.py --gpus 2 --tp 2 --experts 4 --steps 300    # Switch-MoE, experts sharded over 2 GPUs

Task: noisy counting sequences (next token = current + 3 mod vocab, 5 % noise): the loss falls from ln(vocab) towards
the noise floor within a few hundred steps.  Model: Bloom blocks at --hidden/--layers (default 512 / 4, vocab 8192),
bf16, Adam.  Rank 0 prints one line per --every steps and a JSON summary; both arms draw identical batches.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def make_batch(step: int, batch: int, seq: int, vocab: int, dp_rank: int, dp: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(1000 + step)
    start = torch.randint(0, vocab, (batch, 1), generator=g)
    ids = (start + 3 * torch.arange(seq)[None, :]) % vocab
    noise = torch.rand(batch, seq, generator=g) < 0.05
    ids = torch.where(noise, torch.randint(0, vocab, (batch, seq), generator=g), ids)
    return ids.chunk(dp)[dp_rank].contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--every", type=int, default=10)
    ap.add_argument("--tp", type=int, default=0)
    ap.add_argument("--pp", type=int, default=1)
    ap.add_argument("--microbatches", type=int, default=4)
    ap.add_argument("--experts", type=int, default=0)
    ap.add_argument("--moe-every", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=512)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--vocab", type=int, default=8192)
    ap.add_argument("--seq-len", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32, help="global batch (sequences)")
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--hf", action="store_true")
    ap.add_argument("--device", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--out", default=None, help="write the curve (one 'step loss' line per print) to this file")
    args = ap.parse_args()
    bench._env_defaults()
    args.model = "convergence"
    bench.MODEL_SIZES["convergence"] = (args.hidden, args.layers, args.heads, args.vocab)
    tp, pp, dp = bench.layout_of(args)
    args.batch_per_gpu = max(1, args.batch // args.gpus)
    import torch.distributed as dist

    if args.impl == "reference":
        built = bench._build_reference(args)
        if built is None:
            return
        ctx, model, optim, fwd, cfg, (tp, pp, dp), note, dev = built
        from pipegoose.distributed.parallel_mode import ParallelMode as RefMode

        dp_rank = ctx.get_local_rank(RefMode.DATA)
        loss_of = fwd
    else:
        from pipegoose_b200.distributed import ParallelContext, ParallelMode
        from pipegoose_b200.models.bloom import BloomConfig

        BloomConfig.convergence = classmethod(lambda cls: cls(vocab_size=args.vocab, hidden_size=args.hidden,
                                                              n_layer=args.layers, n_head=args.heads))
        ctx = ParallelContext.from_torch(tensor_parallel_size=tp, pipeline_parallel_size=pp, data_parallel_size=dp,
                                         backend="nccl" if args.device == "cuda" else "gloo")
        torch.manual_seed(1234)
        model, optim, cfg = bench._build_ours(args, ctx, torch, hf=args.hf)
        dev = torch.device("cuda", torch.cuda.current_device()) if args.device == "cuda" else torch.device("cpu")
        dp_rank = ctx.get_local_rank(ParallelMode.DATA)
        note = None

        def loss_of(ids):
            return bench._total_loss(model, ids, args.experts)

    rank = ctx.get_global_rank()
    curve = []
    for step in range(args.steps):
        ids = make_batch(step, args.batch, args.seq_len, args.vocab, dp_rank, dp).to(dev)
        loss = loss_of(ids)
        optim.zero_grad()
        loss.backward()
        optim.step()
        if step % args.every == 0 or step == args.steps - 1:
            t = loss.detach().float().clone()
            if dp > 1:   # mean over the data-parallel replicas (every rank of a replica reports the same loss)
                dist.all_reduce(t)
                t /= dist.get_world_size()
            curve.append((step, float(t)))
            if rank == 0:
                print(f"step {step:4d}  loss {float(t):.4f}", flush=True)
    if rank == 0:
        summary = {"impl": args.impl, "parallelism": bench.config_of(args, tp, pp, dp)["parallelism"], "steps": args.steps,
                   "first_loss": curve[0][1], "last_loss": curve[-1][1], "ln_vocab": float(torch.log(torch.tensor(float(args.vocab)))),
                   "converged": curve[-1][1] < 0.5 * curve[0][1], "note": note,
                   "model": {"hidden": args.hidden, "layers": args.layers, "vocab": args.vocab, "seq": args.seq_len,
                             "global_batch": args.batch, "lr": args.lr}}
        print(json.dumps(summary), flush=True)
        if args.out:
            with open(args.out, "w") as f:
                f.write(json.dumps(summary) + "\n")
                for s, l in curve:
                    f.write(f"{s} {l:.5f}\n")
    try:
        if args.impl == "reference":
            dist.barrier()
            dist.destroy_process_group()
        else:
            ctx.destroy()
    except Exception:
        pass


if __name__ == "__main__":
    main()
