"""Times continuous batching: the paged decode-attention kernel against the contiguous one, and ContinuousBatcher
against static batches through generate().

    python tools/serve_bench.py --out profiles/serve_h100.json [--iters 50] [--rounds 2] [--skip-e2e]

Kernel: for B·H in {16, 128, 512} (H = 16), filled length in {512, 2048, 8192, 32768} and D in {64, 128}, one
``alibi_decode_attention`` call on a contiguous ``[B, H, len, D]`` cache and one ``alibi_paged_decode_attention`` call
on the same keys and values spread over shuffled 64-position pages, every row at the same position, are timed with
CUDA events over ``--iters`` launches after warm-up.  Bandwidth follows tools/decode_bench.py: the bytes the kernel
has to move (every visible key and value once, the qkv rows, the output and the cache write) over the time, against
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The page-table reads are not counted.

End to end: random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80), 256 greedy requests with prompts log-uniform
in [16, 1024] tokens and max_new_tokens uniform in [16, 256] (seed 0), all submitted at once.  The engine arm runs them
through one ContinuousBatcher whose pool holds 32 × 1280 positions: the KV memory a static batch of 32 such requests
needs at most.  The static arm runs them in submission order in batches of 32 through generate(): left-padded, every
batch running to its largest max_new_tokens.  Generated tokens/s counts each request's max_new_tokens (not the tokens
a static batch computes past a request's end) over the wall time of the whole set; a request's latency is the time from
the start of the set to the end of the step (engine) or batch (static) that finishes it.  The arms alternate in this
process after one warm-up of each on 16 requests; each arm reports its round with the median wall time (with an even
number of rounds, the fastest), and the wall times of all rounds.

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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decode_bench import HBM_BYTES_PER_S, card, kernel_bytes, time_us  # noqa: E402

STATIC_BATCH = 32
MAX_PROMPT, MAX_NEW = 1024, 256


def kernel_rows(iters: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import PAGE_SIZE, alibi_decode_attention, alibi_paged_decode_attention

    rows = []
    H = 16
    for BH in (16, 128, 512):
        B = BH // H
        for D in (64, 128):
            for length in (512, 2048, 8192, 32768):
                pos = length - 1
                n_pages = length // PAGE_SIZE
                g = torch.Generator(device="cuda").manual_seed(length + D + BH)
                k_cache = torch.randn(B, H, length, D, device="cuda", generator=g, dtype=torch.bfloat16)
                v_cache = torch.randn(B, H, length, D, device="cuda", generator=g, dtype=torch.bfloat16)
                qkv = torch.randn(B, H * 3 * D, device="cuda", generator=g, dtype=torch.bfloat16)
                slopes = K.alibi_slopes(H, device="cuda")
                table = torch.randperm(B * n_pages, device="cuda", generator=g).to(torch.int32).view(B, n_pages)
                k_pool = torch.empty(B * n_pages, H, PAGE_SIZE, D, device="cuda", dtype=torch.bfloat16)
                v_pool = torch.empty_like(k_pool)
                k_pool[table.long()] = k_cache.view(B, H, n_pages, PAGE_SIZE, D).transpose(1, 2)
                v_pool[table.long()] = v_cache.view(B, H, n_pages, PAGE_SIZE, D).transpose(1, 2)
                pos_t = torch.full((B,), pos, dtype=torch.int32, device="cuda")
                want = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, None, D)
                got = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos_t, pos, slopes, D)
                t_cont = time_us(lambda: alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, None, D), iters)
                t_paged = time_us(lambda: alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos_t, pos, slopes,
                                                                        D), iters)
                nbytes = kernel_bytes(B, H, D, pos, None)
                row = {"B": B, "H": H, "BH": BH, "D": D, "len": length,
                       "contiguous_us": round(t_cont, 2), "paged_us": round(t_paged, 2),
                       "paged_over_contiguous": round(t_paged / t_cont, 3), "bytes": nbytes,
                       "contiguous_TBps": round(nbytes / t_cont / 1e6, 3), "paged_TBps": round(nbytes / t_paged / 1e6, 3),
                       "paged_share_of_3.35TBps": round(nbytes / t_paged / 1e6 / (HBM_BYTES_PER_S / 1e12), 3),
                       "bitwise_equal": bool(torch.equal(got, want))}
                print(json.dumps(row), flush=True)
                rows.append(row)
                del k_cache, v_cache, k_pool, v_pool
                torch.cuda.empty_cache()
    return rows


def workload(n: int, seed: int = 0):
    """``n`` requests: prompt lengths log-uniform in [16, MAX_PROMPT], max_new_tokens uniform in [16, MAX_NEW]."""
    import torch

    g = torch.Generator().manual_seed(seed)
    lo, hi = math.log(16), math.log(MAX_PROMPT)
    lengths = [int(round(math.exp(lo + (hi - lo) * u))) for u in torch.rand(n, generator=g).tolist()]
    news = torch.randint(16, MAX_NEW + 1, (n,), generator=g).tolist()
    prompts = [torch.randint(0, 250000, (p,), generator=g).tolist() for p in lengths]
    return prompts, news


def run_engine(model, prompts, news):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=STATIC_BATCH * (MAX_PROMPT + MAX_NEW))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rids = [engine.submit(p, n) for p, n in zip(prompts, news)]
    finish, steps = {}, 0
    while engine.has_work():
        done = engine.step()          # returns after the chosen tokens reached the host: the step is complete
        steps += 1
        now = time.perf_counter()
        for rid, _ in done:
            finish[rid] = now - t0
    return [finish[r] for r in rids], time.perf_counter() - t0, steps


def run_static(model, prompts, news):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lat = []
    for s in range(0, len(prompts), STATIC_BATCH):
        batch, new = prompts[s:s + STATIC_BATCH], news[s:s + STATIC_BATCH]
        P = max(len(p) for p in batch)
        ids = torch.zeros(len(batch), P, dtype=torch.long)
        mask = torch.zeros(len(batch), P, dtype=torch.long)
        for i, p in enumerate(batch):
            ids[i, P - len(p):] = torch.tensor(p)
            mask[i, P - len(p):] = 1
        model.generate(ids.cuda(), max_new_tokens=max(new), attention_mask=mask.cuda())
        torch.cuda.synchronize()
        lat += [time.perf_counter() - t0] * len(batch)
    return lat, time.perf_counter() - t0


def e2e_rows(rounds: int, n_requests: int):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    prompts, news = workload(n_requests)
    warm_p, warm_n = workload(16, seed=1)
    rows = []
    for name, cfg in (("bloom-560m", BloomConfig.bloom_560m()), ("bloom-3b", BloomConfig.bloom_3b())):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = BloomForCausalLM(cfg)
        model = model.to(torch.bfloat16).eval()
        run_engine(model, warm_p, warm_n)
        run_static(model, warm_p, warm_n)
        res = {"engine": [], "static": []}
        for _ in range(rounds):
            lat, wall, steps = run_engine(model, prompts, news)
            res["engine"].append((lat, wall, steps))
            lat, wall = run_static(model, prompts, news)
            res["static"].append((lat, wall, None))
        row = {"model": name, "requests": n_requests, "generated_tokens": sum(news),
               "prompt_tokens": sum(len(p) for p in prompts), "static_batch": STATIC_BATCH,
               "engine_pool_positions": STATIC_BATCH * (MAX_PROMPT + MAX_NEW)}
        for arm, runs in res.items():
            walls = [w for _, w, _ in runs]
            i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
            lat = sorted(runs[i][0])
            row[arm] = {"tokens_per_s": round(sum(news) / walls[i], 1), "wall_s": round(walls[i], 3),
                        "p50_latency_s": round(statistics.median(lat), 3),
                        "p95_latency_s": round(lat[min(len(lat) - 1, int(0.95 * len(lat)))], 3),
                        "wall_s_samples": [round(w, 3) for w in walls]}
            if runs[i][2] is not None:
                row[arm]["steps"] = runs[i][2]
        row["throughput_ratio"] = round(row["engine"]["tokens_per_s"] / row["static"]["tokens_per_s"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="serve_bench.json")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("serve_bench.py measures on a GPU; none is visible")
    result = {"card": card(), "kernel": kernel_rows(args.iters)}
    if not args.skip_e2e:
        result["e2e"] = e2e_rows(args.rounds, args.requests)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
