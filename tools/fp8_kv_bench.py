"""Times the FP8 (e4m3) paged KV cache against the bf16 one: the decode kernel, the cached prefill, and the serving
engine end to end.

    python tools/fp8_kv_bench.py --out profiles/fp8_kv_h100.json [--iters 50] [--rounds 2] [--skip-e2e]

Kernel: the grid of tools/serve_bench.py (B·H in {16, 128, 512} with H = 16, D in {64, 128}, length in {512, 2048,
8192, 32768}, every row at the last position of shuffled 64-position pages).  ``alibi_paged_decode_attention`` on bf16
pools and on the same values quantized into FP8 pools are timed with CUDA events over ``--iters`` launches each,
alternating for ``--rounds`` rounds (the median is kept).  Bytes moved per visible key: ``4·D`` for bf16 (K and V),
``2·(D + 4)`` for FP8 (codes and one fp32 scale each); bandwidth is over the H100 SXM data-sheet 3.35 TB/s.

Cached prefill: 8 sequences of H = 16 heads with a cached prefix of {1024, 8192} positions and {64, 512} new tokens,
D in {64, 128}.  bf16: ``paged_kv_write`` of the new tokens then the paged prefill kernel on the pools.  FP8: the
quantizing ``paged_kv_write`` then the staged prefill (prefix pages dequantized into a bf16 staging pool, new tokens
written into it, the same kernel).  The staging plan is built and uploaded outside the timed region, as the engine
uploads it with the step's other inputs.

End to end: tools/serve_bench.py's workload (256 greedy requests, prompts log-uniform in [16, 1024], max_new_tokens
uniform in [16, 256], seed 0) on random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80), three ContinuousBatcher
arms alternated after a warm-up: bf16 pools of 40960 positions, FP8 pools of the same bytes (40960·2D / (D + 4)
positions, about 1.9×), and FP8 pools of 40960 positions (the kernels without the capacity).  Each reports tokens/s,
p50 / p95 latency, steps and the most requests decoding at once, from its median round.

Logit deviation: the FP8 engine teacher-forced with the bf16 engine's tokens on 16 requests of the same workload; the
largest |logit difference| per step over that step's max |logit|.  The models are random-init: this measures the
arithmetic, it is not a claim about quality on trained weights.

The card name and power limit are read in the same run and written next to the numbers."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decode_bench import HBM_BYTES_PER_S, card, time_us  # noqa: E402
from serve_bench import MAX_NEW, MAX_PROMPT, STATIC_BATCH, workload  # noqa: E402

FP8 = None   # torch.float8_e4m3fn, set in main()
BF16_POSITIONS = STATIC_BATCH * (MAX_PROMPT + MAX_NEW)


def _quantized(pool):
    """``pool`` quantized page block by page block (bounded temporaries): (codes, scales)."""
    import torch

    from pipegoose_b200.ops.attention import quantize_kv

    codes = torch.empty(pool.shape, dtype=FP8, device=pool.device)
    scales = torch.empty(pool.shape[:-1], dtype=torch.float32, device=pool.device)
    for i in range(0, pool.shape[0], 1024):
        codes[i:i + 1024], scales[i:i + 1024] = quantize_kv(pool[i:i + 1024])
    return codes, scales


def _alternate(fns, iters, rounds):
    times = [[] for _ in fns]
    for _ in range(rounds):
        for t, fn in zip(times, fns):
            t.append(time_us(fn, iters))
    return [statistics.median(t) for t in times]


def kernel_rows(iters: int, rounds: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import PAGE_SIZE, alibi_paged_decode_attention

    rows = []
    H = 16
    for BH in (16, 128, 512):
        B = BH // H
        for D in (64, 128):
            for length in (512, 2048, 8192, 32768):
                pos = length - 1
                n_pages = length // PAGE_SIZE
                g = torch.Generator(device="cuda").manual_seed(length + D + BH)
                k_pool = torch.randn(B * n_pages, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
                v_pool = torch.randn(B * n_pages, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
                table = torch.randperm(B * n_pages, device="cuda", generator=g).to(torch.int32).view(B, n_pages)
                qkv = torch.randn(B, H * 3 * D, device="cuda", generator=g, dtype=torch.bfloat16)
                slopes = K.alibi_slopes(H, device="cuda")
                pos_t = torch.full((B,), pos, dtype=torch.int32, device="cuda")
                k8, ks = _quantized(k_pool)
                v8, vs = _quantized(v_pool)
                want = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos_t, pos, slopes, D)
                got = alibi_paged_decode_attention(qkv, k8, v8, table, pos_t, pos, slopes, D, k_scales=ks, v_scales=vs)
                t16, t8 = _alternate([
                    lambda: alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos_t, pos, slopes, D),
                    lambda: alibi_paged_decode_attention(qkv, k8, v8, table, pos_t, pos, slopes, D, k_scales=ks,
                                                         v_scales=vs)], iters, rounds)
                keys = B * H * (pos + 1)
                b16, b8 = keys * 4 * D, keys * 2 * (D + 4)
                row = {"B": B, "H": H, "BH": BH, "D": D, "len": length,
                       "bf16_us": round(t16, 2), "fp8_us": round(t8, 2), "speedup": round(t16 / t8, 3),
                       "bf16_bytes": b16, "fp8_bytes": b8,
                       "bf16_TBps": round(b16 / t16 / 1e6, 3), "fp8_TBps": round(b8 / t8 / 1e6, 3),
                       "bf16_share_of_3.35TBps": round(b16 / t16 / 1e6 / (HBM_BYTES_PER_S / 1e12), 3),
                       "fp8_share_of_3.35TBps": round(b8 / t8 / 1e6 / (HBM_BYTES_PER_S / 1e12), 3),
                       "fp8_vs_bf16_rel_err": round(((got.float() - want.float()).abs().max()
                                                     / want.float().abs().max()).item(), 4)}
                print(json.dumps(row), flush=True)
                rows.append(row)
                del k_pool, v_pool, k8, v8, ks, vs
                torch.cuda.empty_cache()
    return rows


def prefill_rows(iters: int, rounds: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_paged_prefill_attention, fp8_prefill_staging,
                                              paged_kv_write)

    rows = []
    R, H = 8, 16
    for D in (64, 128):
        for prefix in (1024, 8192):
            for new in (64, 512):
                total = prefix + new
                per = -(-total // PAGE_SIZE)
                g = torch.Generator(device="cuda").manual_seed(prefix + new + D)
                k_pool = torch.randn(R * per, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
                v_pool = torch.randn(R * per, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
                k8, ks = _quantized(k_pool)
                v8, vs = _quantized(v_pool)
                perm = torch.randperm(R * per, generator=torch.Generator().manual_seed(D)).tolist()
                pages = [perm[r * per:(r + 1) * per] for r in range(R)]
                dev = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
                table = dev(pages)
                slot = dev([pages[r][p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE
                            for r in range(R) for p in range(prefix, total)])
                cu = dev([r * new for r in range(R + 1)])
                start = dev([prefix] * R)
                qkv = torch.randn(R * new, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
                slopes = K.alibi_slopes(H, device="cuda")
                n, src, dst, st_slot, st_table = fp8_prefill_staging(pages, [prefix] * R, [total] * R)
                k_st = torch.empty(n, H, PAGE_SIZE, D, device="cuda", dtype=torch.bfloat16)
                stage = (k_st, torch.empty_like(k_st), dev(src), dev(dst), dev(st_slot), dev(st_table))

                def bf16():
                    paged_kv_write(qkv, slot, k_pool, v_pool, D)
                    return alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, new, slopes, D)

                def fp8():
                    paged_kv_write(qkv, slot, k8, v8, D, k_scales=ks, v_scales=vs)
                    return alibi_paged_prefill_attention(qkv, k8, v8, table, cu, start, new, slopes, D, k_scales=ks,
                                                         v_scales=vs, stage=stage)

                want, got = bf16(), fp8()
                t16, t8 = _alternate([bf16, fp8], iters, rounds)
                row = {"R": R, "H": H, "D": D, "prefix": prefix, "new": new, "bf16_us": round(t16, 2),
                       "fp8_staged_us": round(t8, 2), "fp8_over_bf16": round(t8 / t16, 3),
                       "fp8_vs_bf16_rel_err": round(((got.float() - want.float()).abs().max()
                                                     / want.float().abs().max()).item(), 4)}
                print(json.dumps(row), flush=True)
                rows.append(row)
                del k_pool, v_pool, k8, v8, ks, vs, stage, k_st
                torch.cuda.empty_cache()
    return rows


def run_engine(model, prompts, news, positions, dtype):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=positions, kv_cache_dtype=dtype)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rids = [engine.submit(p, n) for p, n in zip(prompts, news)]
    finish, steps, peak = {}, 0, 0
    while engine.has_work():
        done = engine.step()
        steps += 1
        peak = max(peak, len(engine._running) + len(done))
        now = time.perf_counter()
        for rid, _ in done:
            finish[rid] = now - t0
    return [finish[r] for r in rids], time.perf_counter() - t0, steps, peak


def deviation(model, prompts, news):
    """Teacher-forced: the FP8 engine takes the bf16 engine's tokens; per decode step, max |diff| / max |logit|."""
    from pipegoose_b200.serving import ContinuousBatcher

    logits, picks = {}, {}
    for dtype in (None, FP8):
        engine = ContinuousBatcher(model, max_cache_tokens=BF16_POSITIONS, kv_cache_dtype=dtype)
        forward, select = engine._forward, engine._select

        def spy(forward=forward, dtype=dtype):
            reqs, out = forward()
            for j, r in enumerate(reqs):
                logits[(dtype, r.rid, len(r.tokens))] = out[j].clone()
            return reqs, out
        engine._forward = spy
        if dtype is None:
            def lead(reqs, out, select=select):
                chosen = select(reqs, out)
                picks.update({(r.rid, len(r.tokens)): t for r, t in zip(reqs, chosen)})
                return chosen
            engine._select = lead
        else:
            engine._select = lambda reqs, out: [picks[(r.rid, len(r.tokens))] for r in reqs]
        for p, n in zip(prompts, news):
            engine.submit(p, n)
        engine.run()
    dist = []
    for (dtype, rid, n), l16 in logits.items():
        if dtype is None and n > len(prompts[rid]):      # decode steps (the prefills are bitwise equal)
            l8 = logits[(FP8, rid, n)]
            dist.append(((l8 - l16).abs().max() / l16.abs().max()).item())
    firsts = all(bool((logits[(FP8, r, len(prompts[r]))] == logits[(None, r, len(prompts[r]))]).all())
                 for r in range(len(prompts)))
    return {"steps": len(dist), "max": round(max(dist), 4), "median": round(statistics.median(dist), 4),
            "prefill_logits_bitwise_equal": firsts}


def e2e_rows(rounds: int, n_requests: int):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    prompts, news = workload(n_requests)
    warm_p, warm_n = workload(16, seed=1)
    dev_p, dev_n = workload(16, seed=2)
    rows = []
    for name, cfg in (("bloom-560m", BloomConfig.bloom_560m()), ("bloom-3b", BloomConfig.bloom_3b())):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = BloomForCausalLM(cfg)
        model = model.to(torch.bfloat16).eval()
        D = cfg.hidden_size // cfg.n_head
        arms = {"bf16": (BF16_POSITIONS, None), "fp8_same_bytes": (BF16_POSITIONS * 2 * D // (D + 4), FP8),
                "fp8_same_positions": (BF16_POSITIONS, FP8)}
        for positions, dtype in arms.values():
            run_engine(model, warm_p, warm_n, positions, dtype)
        res = {arm: [] for arm in arms}
        for _ in range(rounds):
            for arm, (positions, dtype) in arms.items():
                res[arm].append(run_engine(model, prompts, news, positions, dtype))
        row = {"model": name, "D": D, "requests": n_requests, "generated_tokens": sum(news),
               "prompt_tokens": sum(len(p) for p in prompts)}
        for arm, runs in res.items():
            walls = [w for _, w, _, _ in runs]
            i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
            lat = sorted(runs[i][0])
            row[arm] = {"pool_positions": arms[arm][0] // 64 * 64, "tokens_per_s": round(sum(news) / walls[i], 1),
                        "wall_s": round(walls[i], 3), "p50_latency_s": round(statistics.median(lat), 3),
                        "p95_latency_s": round(lat[min(len(lat) - 1, int(0.95 * len(lat)))], 3),
                        "steps": runs[i][2], "peak_running": runs[i][3],
                        "wall_s_samples": [round(w, 3) for w in walls]}
        row["logit_deviation_random_init_not_a_quality_claim"] = deviation(model, dev_p, dev_n)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    global FP8
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="fp8_kv_bench.json")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("fp8_kv_bench.py measures on a GPU; none is visible")
    FP8 = torch.float8_e4m3fn
    result = {"card": card(), "kernel": kernel_rows(args.iters, args.rounds),
              "cached_prefill": prefill_rows(args.iters, args.rounds)}
    if not args.skip_e2e:
        result["e2e"] = e2e_rows(args.rounds, args.requests)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
