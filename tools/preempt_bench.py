"""Measures preemption in ContinuousBatcher: the swap kernel's rate and serving throughput with pages taken as
sequences grow.

    python tools/preempt_bench.py --out profiles/preempt_h100.json [--requests 64] [--rounds 2]

(a) ``paged_kv_swap`` on bloom-560m's pool shape (24 layers, 16 heads, 64 positions, D = 64), bf16 and FP8 (codes and
scales), 1 .. 512 pages at scattered page and slot ids, to the host and back, timed with CUDA events (median of 5
rounds).  Reported: GB/s of the bytes moved, against one ``cudaMemcpyAsync`` (``Tensor.copy_(non_blocking=True)``) of
a contiguous pinned buffer of the same byte count in the same direction: the copy engine's rate, the ceiling for
this traffic.

(b) Random-init bf16 bloom-560m with a 64-token vocabulary (its greedy outputs repeat one token, so a greedy eos
workload stops every request after one token; over 64 tokens its distribution is near uniform) serving ``--requests``
sampled requests (prompts log-uniform in [16, 512], ``max_new_tokens = 512``, all stopping at ``eos_token_id`` = 7
if they sample it first) from a 256-page pool (16384 positions) that cannot hold every request's worst case.  Three
engines: reservation (``preemption=False``), ``preemption=True`` with ``swap_space_tokens=0`` (recompute only) and
with a host pool as large as the device pool, each with the same seeded generator.  Sampled tokens depend on which
requests share a step, so the engines' outputs are compared by their generated-length distribution, not token for
token.  Arms alternate over ``--rounds`` rounds after a warm-up; reported per arm: generated tokens / s (median wall
time; with an even number of rounds the fastest), mean running rows per decode step and the preemption counters.

The card name and power limit are read in the same run and written next to the numbers."""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decode_bench import card  # noqa: E402

LAYERS, HEADS, D = 24, 16, 64                  # bloom-560m
PAGES = (1, 4, 16, 64, 256, 512)
POOL_PAGES = 256
MAX_NEW = 512


def _events_ms(fn, iters):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def swap_rows():
    import torch

    from pipegoose_b200.ops.attention import PAGE_SIZE, paged_kv_swap

    n_max = max(PAGES)
    shape = (LAYERS, n_max, HEADS, PAGE_SIZE, D)
    page_bytes = LAYERS * 2 * HEADS * PAGE_SIZE * D * 2                       # bf16 K and V of one page
    buf = torch.empty(n_max * page_bytes, dtype=torch.uint8).pin_memory()   # host pool of either dtype, and the ceiling
    dev = torch.empty(n_max * page_bytes, dtype=torch.uint8, device="cuda")
    g = torch.Generator().manual_seed(0)
    rows = []
    for fp8 in (False, True):
        k = torch.randn(shape, device="cuda").to(torch.float8_e4m3fn if fp8 else torch.bfloat16)
        v = torch.randn(shape, device="cuda").to(k.dtype)
        ks = vs = hs = None
        host_shape = (n_max, LAYERS, 2, HEADS, PAGE_SIZE, D)
        kv_bytes = math.prod(host_shape) * k.element_size()
        host = buf[:kv_bytes].view(k.dtype).view(host_shape)
        if fp8:
            ks, vs = torch.rand(shape[:-1], device="cuda"), torch.rand(shape[:-1], device="cuda")
            hs = buf[kv_bytes:kv_bytes + math.prod(host_shape[:-1]) * 4].view(torch.float32).view(host_shape[:-1])
        for n in PAGES:
            pairs = torch.stack([torch.randperm(n_max, generator=g)[:n], torch.randperm(n_max, generator=g)[:n]], 1)
            pairs = pairs.to(torch.int32).cuda()
            nbytes = n * (page_bytes // (2 if fp8 else 1) + (LAYERS * 2 * HEADS * PAGE_SIZE * 4 if fp8 else 0))
            iters = max(3, min(200, (2 << 30) // nbytes))
            row = {"pools": "fp8" if fp8 else "bf16", "pages": n, "bytes": nbytes}
            for to_host in (True, False):
                def swap():
                    paged_kv_swap(pairs, k, v, ks, vs, host, hs, to_host)

                def memcpy():
                    (buf[:nbytes].copy_(dev[:nbytes], non_blocking=True) if to_host
                     else dev[:nbytes].copy_(buf[:nbytes], non_blocking=True))

                swap(), memcpy()
                t_swap, t_copy = [], []
                for _ in range(5):                                   # the two arms alternate
                    t_swap.append(_events_ms(swap, iters))
                    t_copy.append(_events_ms(memcpy, iters))
                ms, mc = statistics.median(t_swap), statistics.median(t_copy)
                key = "to_host" if to_host else "from_host"
                row[key] = {"swap_ms": round(ms, 4), "swap_GBps": round(nbytes / ms / 1e6, 2),
                            "memcpy_ms": round(mc, 4), "memcpy_GBps": round(nbytes / mc / 1e6, 2),
                            "swap_over_memcpy": round(mc / ms, 3)}
            print(json.dumps(row), flush=True)
            rows.append(row)
        del k, v, ks, vs
    del buf, dev
    torch.cuda.empty_cache()
    return rows


VOCAB, EOS = 64, 7


def workload(n, seed=0):
    import torch

    g = torch.Generator().manual_seed(seed)
    lo, hi = math.log(16), math.log(512)
    lengths = [int(round(math.exp(lo + (hi - lo) * u))) for u in torch.rand(n, generator=g).tolist()]
    return [torch.randint(0, VOCAB, (p,), generator=g).tolist() for p in lengths]


def run(model, prompts, **kw):
    """One engine over every request (all submitted at once); returns the generated lengths, wall seconds, mean
    running rows per decode step and the counters."""
    import torch

    from pipegoose_b200.ops.attention import PAGE_SIZE
    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=kw.pop("pages", POOL_PAGES) * PAGE_SIZE,
                               generator=torch.Generator(device="cuda").manual_seed(0), **kw)
    rows = []
    forward = engine._forward

    def spy():
        if not engine._admitted:
            rows.append(len(engine._running))
        return forward()

    engine._forward = spy
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rids = [engine.submit(p, MAX_NEW, do_sample=True, eos_token_id=EOS) for p in prompts]
    outs = engine.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    counters = {k: getattr(engine, k) for k in ("preemptions", "swapped_out_pages", "swapped_in_pages",
                                                "recomputed_tokens")}
    return [len(outs[r]) - len(p) for r, p in zip(rids, prompts)], wall, sum(rows) / max(1, len(rows)), counters


def serving(n_requests, rounds):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.ops.attention import PAGE_SIZE

    torch.manual_seed(0)
    cfg = BloomConfig.bloom_560m()
    cfg.vocab_size = VOCAB
    with torch.device("cuda"):
        model = BloomForCausalLM(cfg)
    model = model.to(torch.bfloat16).eval()
    prompts = workload(n_requests)
    arms = {"reservation": {}, "recompute": dict(preemption=True),
            "swap": dict(preemption=True, swap_space_tokens=POOL_PAGES * PAGE_SIZE)}
    warm = workload(8, seed=1)
    for kw in arms.values():
        run(model, warm, **dict(kw, pages=64))
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, kw in arms.items():
            res[name].append(run(model, prompts, **dict(kw)))
            print(name, round(res[name][-1][1], 3), flush=True)
    out = {"model": f"bloom-560m geometry, vocabulary {VOCAB} (random init, bf16)", "requests": n_requests,
           "max_new_tokens": MAX_NEW, "eos_token_id": EOS, "sampling": "do_sample=True, temperature 1",
           "pool_pages": POOL_PAGES, "pool_positions": POOL_PAGES * PAGE_SIZE,
           "worst_case_pages": sum(-(-(len(p) + MAX_NEW) // PAGE_SIZE) for p in prompts),
           "host_pool_pages_swap_arm": POOL_PAGES}
    for name, runs in res.items():
        walls = [r[1] for r in runs]
        i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
        lens, wall, rows, counters = runs[i]
        out[name] = {"tokens_per_s": round(sum(lens) / wall, 1), "generated_tokens": sum(lens),
                     "mean_generated_length": round(statistics.mean(lens), 1),
                     "median_generated_length": statistics.median(lens), "wall_s": round(wall, 3),
                     "wall_s_samples": [round(w, 3) for w in walls], "mean_running_rows_per_decode_step": round(rows, 2),
                     **counters}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="preempt_bench.json")
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-serving", action="store_true")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("preempt_bench measures on the GPU: no CUDA device")
    res = {"card": card(), "swap_kernel": swap_rows()}
    if not args.skip_serving:
        res["serving"] = serving(args.requests, args.rounds)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
