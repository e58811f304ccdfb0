"""Times prefix caching: the paged prefill-attention kernel, and ContinuousBatcher with prefix_caching on and off.

    python tools/prefix_bench.py --out profiles/prefix_h100.json [--iters 30] [--rounds 2] [--skip-e2e]

Kernel: H = 16, D in {64, 80, 128}, 8 sequences, each with (cached prefix, new tokens) in {(0, 512), (0, 2048),
(1024, 64), (1024, 256), (4096, 512), (8192, 128)}, keys and values on shuffled 64-position pages.  One
``alibi_paged_prefill_attention`` call is timed with CUDA events over ``--iters`` launches after warm-up.  Useful work
counts the visible (query, key) pairs, 4·D flops each (Q·K and P·V), against the H100 SXM data-sheet dense BF16 rate
(989 TFLOP/s).  For the start = 0 rows the document-masked flash kernel (``alibi_attention`` with ``seg_start``) runs on
the same packed tokens with keys from qkv; ``paged_over_flash`` is the cost of reading K / V through pages.  At D = 80
the flash path pads Q / K / V to 128 columns and back around the kernel, and that copy is inside its time.

End to end: random-init bf16 bloom-560m and bloom-3b, 256 greedy requests, each one of 4 system prompts of 1024 tokens
followed by a unique suffix log-uniform in [16, 256] tokens, max_new_tokens uniform in [16, 128] (seed 0), all
submitted at once into a pool of 32 × 1408 positions.  The two arms (prefix_caching on / off, same pool) alternate in
this process after one warm-up of each on 16 requests; each arm reports its round with the median wall time (with an
even number of rounds, the fastest): generated tokens/s, p50 / p95 finish latency, the summed wall time of the prefill
steps, and prompt tokens computed against served from the cache.

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
from decode_bench import card, time_us  # noqa: E402

PEAK_BF16_FLOPS = 989e12
SHAPES = [(0, 512), (0, 2048), (1024, 64), (1024, 256), (4096, 512), (8192, 128)]
SYSTEM, SUFFIX, MAX_NEW, POOL = 1024, 256, 128, 32 * 1408


def kernel_rows(iters: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_attention, alibi_paged_prefill_attention,
                                              paged_kv_write)

    rows = []
    H, R = 16, 8
    for D in (64, 80, 128):
        for st, n in SHAPES:
            g = torch.Generator(device="cuda").manual_seed(st + n + D)
            need = (st + n - 1) // PAGE_SIZE + 1
            table = torch.randperm(R * need, device="cuda", generator=g).to(torch.int32).view(R, need)
            k_pool = torch.randn(R * need, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
            v_pool = torch.randn_like(k_pool)
            qkv = torch.randn(R * n, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
            cu = torch.arange(0, R * n + 1, n, dtype=torch.int32, device="cuda")
            start = torch.full((R,), st, dtype=torch.int32, device="cuda")
            slopes = K.alibi_slopes(H, device="cuda")
            if st == 0:        # the new tokens' keys in their slots, as the engine stores them
                p = torch.arange(n, device="cuda").repeat(R)
                slot = (table[torch.arange(R, device="cuda").repeat_interleave(n), p // PAGE_SIZE] * PAGE_SIZE
                        + p % PAGE_SIZE).to(torch.int32)
                paged_kv_write(qkv, slot, k_pool, v_pool, D)
            t_paged = time_us(lambda: alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, n, slopes,
                                                                    D), iters)
            pairs = R * (n * st + n * (n + 1) // 2)
            flops = 4 * D * H * pairs
            row = {"H": H, "D": D, "sequences": R, "cached": st, "new": n, "paged_us": round(t_paged, 2),
                   "visible_pairs_per_head": pairs, "TFLOPs": round(flops / t_paged / 1e6, 1),
                   "share_of_989": round(flops / t_paged / 1e6 / (PEAK_BF16_FLOPS / 1e12), 3)}
            if st == 0:
                seg = torch.arange(R, device="cuda", dtype=torch.int32).repeat_interleave(n).mul(n).view(1, R * n)
                with torch.no_grad():
                    t_flash = time_us(lambda: alibi_attention(qkv, slopes, 1, R * n, H, D, seg_start=seg), iters)
                    want = alibi_attention(qkv, slopes, 1, R * n, H, D, seg_start=seg)
                got = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, n, slopes, D)
                row.update({"flash_us": round(t_flash, 2), "paged_over_flash": round(t_paged / t_flash, 3),
                            "max_abs_diff_vs_flash": float((got.float() - want.float()).abs().max()),
                            "flash_includes_padding_copies": D == 80})
            print(json.dumps(row), flush=True)
            rows.append(row)
            del k_pool, v_pool, qkv
            torch.cuda.empty_cache()
    return rows


def workload(n: int, seed: int = 0):
    """``n`` requests: one of 4 system prompts of SYSTEM tokens + a unique suffix log-uniform in [16, SUFFIX],
    max_new_tokens uniform in [16, MAX_NEW]."""
    import torch

    g = torch.Generator().manual_seed(seed)
    systems = [torch.randint(0, 250000, (SYSTEM,), generator=g).tolist() for _ in range(4)]
    lo, hi = math.log(16), math.log(SUFFIX)
    lengths = [int(round(math.exp(lo + (hi - lo) * u))) for u in torch.rand(n, generator=g).tolist()]
    which = torch.randint(0, 4, (n,), generator=g).tolist()
    news = torch.randint(16, MAX_NEW + 1, (n,), generator=g).tolist()
    prompts = [systems[w] + torch.randint(0, 250000, (p,), generator=g).tolist() for w, p in zip(which, lengths)]
    return prompts, news


def run_engine(model, prompts, news, prefix_caching: bool):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=POOL, prefix_caching=prefix_caching)
    forward, kind = engine._forward, []

    def spy():
        kind.append(bool(engine._admitted))          # a step with admitted prompts is a prefill step
        return forward()

    engine._forward = spy
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rids = [engine.submit(p, n) for p, n in zip(prompts, news)]
    finish, prefill_s = {}, 0.0
    while engine.has_work():
        s0 = time.perf_counter()
        done = engine.step()          # returns after the chosen tokens reached the host: the step is complete
        now = time.perf_counter()
        if kind and kind[-1]:
            prefill_s += now - s0
        kind.clear()
        for rid, _ in done:
            finish[rid] = now - t0
    return [finish[r] for r in rids], time.perf_counter() - t0, prefill_s, engine.cached_prompt_tokens


def e2e_rows(rounds: int, n_requests: int):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    prompts, news = workload(n_requests)
    warm_p, warm_n = workload(16, seed=1)
    prompt_tokens = sum(len(p) for p in prompts)
    rows = []
    for name, cfg in (("bloom-560m", BloomConfig.bloom_560m()), ("bloom-3b", BloomConfig.bloom_3b())):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = BloomForCausalLM(cfg)
        model = model.to(torch.bfloat16).eval()
        run_engine(model, warm_p, warm_n, True)
        run_engine(model, warm_p, warm_n, False)
        res = {"prefix_caching": [], "no_prefix_caching": []}
        for _ in range(rounds):
            res["prefix_caching"].append(run_engine(model, prompts, news, True))
            res["no_prefix_caching"].append(run_engine(model, prompts, news, False))
        row = {"model": name, "requests": n_requests, "generated_tokens": sum(news), "prompt_tokens": prompt_tokens,
               "pool_positions": POOL}
        for arm, runs in res.items():
            walls = [r[1] for r in runs]
            i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
            lat, wall, prefill_s, cached = runs[i]
            lat = sorted(lat)
            row[arm] = {"tokens_per_s": round(sum(news) / wall, 1), "wall_s": round(wall, 3),
                        "p50_latency_s": round(statistics.median(lat), 3),
                        "p95_latency_s": round(lat[min(len(lat) - 1, int(0.95 * len(lat)))], 3),
                        "prefill_steps_s": round(prefill_s, 3), "prompt_tokens_computed": prompt_tokens - cached,
                        "prompt_tokens_cached": cached, "wall_s_samples": [round(w, 3) for w in walls]}
        row["throughput_ratio"] = round(row["prefix_caching"]["tokens_per_s"] / row["no_prefix_caching"]["tokens_per_s"],
                                        3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="prefix_bench.json")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("prefix_bench.py measures on a GPU; none is visible")
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
