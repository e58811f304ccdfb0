"""Fused TP kernels vs NCCL + plain GEMM at model shapes.  torchrun --nproc-per-node T tools/tp_bench.py
Writes gpurun_out/tp_bench_T{T}.json (rank 0).  Times are CUDA-event, max over ranks."""
import json, os, sys
import torch, torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipegoose_b200.distributed import ParallelContext, ParallelMode
from pipegoose_b200.parallel.tp_comm import TensorParallelComm
from pipegoose_b200.ops import kernels as K
from pipegoose_b200.constants import H100_BF16_DENSE_FLOPS, H100_NVLINK_BYTES_PER_S

T = int(os.environ["WORLD_SIZE"])
ctx = ParallelContext.from_torch(tensor_parallel_size=T, pipeline_parallel_size=1, data_parallel_size=1, backend="nccl")
dev = torch.device("cuda", torch.cuda.current_device())
comm = TensorParallelComm(ctx, fused=True); comm.enable_fused()
rank = ctx.get_global_rank()

def timeit(fn, iters=20):
    for _ in range(5): fn()
    torch.cuda.synchronize(); dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()

model = os.environ.get("TPB_MODEL", "560m")
h, seq, b = {"560m": (1024, 1024, 8 * T), "7b1": (4096, 2048, 8)}[model]
M = b * seq
rows = []
for name, kind, N, Kd in [("qkv", "ag", 3 * h // T, h), ("fc1", "ag", 4 * h // T, h), ("dense", "rs", h, h // T), ("fc2", "rs", h, 4 * h // T)]:
    torch.manual_seed(1)
    if kind == "ag":
        x = torch.randn(M // T, Kd, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16) * 0.02
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
        fused = timeit(lambda: comm.ag_gemm(x, w, bias))
        lib = timeit(lambda: K.gemm_nt(comm.all_gather_rows(x), w, bias))
        xf = comm.all_gather_rows(x)
        gemm_only = timeit(lambda: K.gemm_nt(xf, w, bias))
        coll_only = timeit(lambda: comm.all_gather_rows(x))
        nvl_bytes = (T - 1) * (M // T) * Kd * 2
    else:
        a = torch.randn(M, Kd, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16) * 0.02
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
        res = torch.randn(M // T, N, device=dev, dtype=torch.bfloat16)
        fused = timeit(lambda: comm.gemm_rs(a, w, bias, res))
        lib = timeit(lambda: comm.reduce_scatter_rows(K.gemm_nt(a, w)) + bias + res)
        gemm_only = timeit(lambda: K.gemm_nt(a, w))
        part = K.gemm_nt(a, w)
        coll_only = timeit(lambda: comm.reduce_scatter_rows(part))
        nvl_bytes = (T - 1) * (M // T) * N * 2
    flops = 2.0 * M * N * Kd
    t_flops = flops / H100_BF16_DENSE_FLOPS * 1e3   # ms at the data-sheet dense bf16 peak
    t_link = nvl_bytes / H100_NVLINK_BYTES_PER_S * 1e3    # ms at the data-sheet NVLink bandwidth per direction
    roof = max(t_flops, t_link)
    rows.append(dict(op=name, kind=kind, M=M, N=N, K=Kd, T=T, fused_ms=fused, nccl_plus_gemm_ms=lib, gemm_only_ms=gemm_only,
                     collective_only_ms=coll_only, roofline_ms=roof, fused_frac_of_roofline=roof / fused,
                     bound="link" if t_link > t_flops else "compute"))
    if rank == 0:
        print(json.dumps(rows[-1]), flush=True)
if rank == 0:
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(rows, open(f"gpurun_out/tp_bench_{model}_T{T}.json", "w"), indent=1)
ctx.destroy()
