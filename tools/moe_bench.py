"""Fused Switch-MoE layer (router kernel + NVLink dispatch + grouped wgmma GEMMs + scatter-combine epilogue) against
the reference-style layer (replicated tokens, per-expert GEMMs, all-reduce combine) at bloom-560m shapes —
BASELINE.json config #4.  (Written without GPU access; first run is its own validation.)

    torchrun --nnodes=1 --nproc-per-node T --master-addr 127.0.0.1 tools/moe_bench.py [--experts 8] [--tokens-per-rank 8192]

Times are CUDA-event, max over ranks; the roofline of the fused layer is the slower of the expert FLOPs at the H100
data-sheet dense bf16 peak and the dispatch + combine bytes over NVLink at its data-sheet 450 GB/s per direction.  Rank 0
prints the result as one JSON line and, with --out PATH, also writes it to PATH.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipegoose_b200.constants import H100_BF16_DENSE_FLOPS, H100_NVLINK_BYTES_PER_S  # noqa: E402
from pipegoose_b200.distributed import ParallelContext  # noqa: E402
from pipegoose_b200.models.bloom import BloomConfig, BloomMLP  # noqa: E402
from pipegoose_b200.nn.expert_parallel import SwitchNoisePolicy, Top1Router, Top2Router  # noqa: E402
from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer  # noqa: E402
from pipegoose_b200.ops.moe import FusedExpertLayer  # noqa: E402


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--experts", type=int, default=8)
    ap.add_argument("--top-k", type=int, default=1)
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--tokens-per-rank", type=int, default=8192)
    ap.add_argument("--out", default=None, help="also write the result JSON to this path (rank 0)")
    args = ap.parse_args()
    T = int(os.environ["WORLD_SIZE"])
    ctx = ParallelContext.from_torch(tensor_parallel_size=T, pipeline_parallel_size=1, data_parallel_size=1, backend="nccl")
    rank = ctx.get_global_rank()
    dev = torch.device("cuda", torch.cuda.current_device())
    h, n, E, k = args.hidden, args.tokens_per_rank, args.experts, args.top_k
    torch.manual_seed(0)
    cfg = BloomConfig(hidden_size=h, n_layer=1, n_head=16)
    expert = BloomMLP(cfg).to(torch.bfloat16).to(dev)
    router_cls = Top1Router if k == 1 else Top2Router

    def router():
        torch.manual_seed(1)
        return router_cls(SwitchNoisePolicy(), E, h, expert_capacity=(1.25, 2.0)).to(torch.bfloat16).to(dev)

    fused = FusedExpertLayer(E, expert, router(), ctx).to(dev)
    plain = ExpertLayer(E, expert, router(), False, ctx).to(dev)
    fused.train(), plain.train()

    torch.manual_seed(100 + rank)
    x_local = torch.randn(n, h, device=dev, dtype=torch.bfloat16, requires_grad=True)   # token-sharded (fused path)
    res_local = torch.randn(n, h, device=dev, dtype=torch.bfloat16)
    x_full = torch.randn(n * T, h, device=dev, dtype=torch.bfloat16, requires_grad=True)  # replicated tokens (reference-style)
    res_full = torch.randn(n * T, h, device=dev, dtype=torch.bfloat16)

    def run_fused():
        y = fused(x_local, res_local)
        y.float().pow(2).mean().backward()

    def run_plain():
        y = plain(x_full.view(1, n * T, h), res_full.view(1, n * T, h))
        y.float().pow(2).mean().backward()

    t_fused = timeit(run_fused)
    t_plain = timeit(run_plain)
    # roofline of the fused layer (forward + backward): expert GEMMs 3 x (2 GEMMs x 2 n k h 4h) and four all-to-alls
    flops = 3 * 2 * 2.0 * n * k * h * 4 * h
    nvl_bytes = 4 * n * k * h * 2 * (T - 1) / T
    roof_ms = max(flops / H100_BF16_DENSE_FLOPS, nvl_bytes / H100_NVLINK_BYTES_PER_S) * 1e3
    row = dict(T=T, experts=E, top_k=k, tokens_per_rank=n, hidden=h, fused_ms=t_fused, reference_style_ms=t_plain,
               roofline_ms=roof_ms, fused_frac_of_roofline=roof_ms / t_fused,
               bound="link" if nvl_bytes / H100_NVLINK_BYTES_PER_S > flops / H100_BF16_DENSE_FLOPS else "compute",
               note="reference-style layer processes T x the tokens per rank (replicated activations) and combines with an all-reduce")
    if rank == 0:
        print(json.dumps(row), flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(row, f, indent=1)
    ctx.destroy()


if __name__ == "__main__":
    main()
