"""Times the serving engine's inter-token gaps with and without chunked prefill while long prompts arrive.

    python tools/chunked_bench.py --out profiles/chunked_prefill_h100.json [--rounds 3] [--chunk 1024]

Random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80), pools of bf16 or FP8, chunking off (the default
``max_prefill_tokens`` = 8192: a longer prompt runs alone) or on (``max_prefill_tokens`` = ``--chunk``).  A steady
decode load of 64 greedy requests (prompts of 32 tokens, 256 new tokens each) runs while four long prompts of 4096,
8192, 12288 and 16384 tokens (16 new tokens each) arrive, one every 24 steps from step 24.  Reported: p50 / p99 /
max gap between consecutive tokens of the 64 decoding requests (host clock per step; every step ends in a
device-to-host transfer), the long prompts' time to first token, generated tokens per second and steps.  The arms of
a model are alternated for ``--rounds`` rounds after a warm-up run; each metric is the median over rounds, with the
p99 gap's and tokens/s's range over rounds next to it and every round's numbers in ``rounds``.

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
from decode_bench import card  # noqa: E402

SHORT, SHORT_PROMPT, SHORT_NEW = 64, 32, 256
LONG = (4096, 8192, 12288, 16384)
LONG_NEW, LONG_EVERY = 16, 24


def run_engine(model, dtype, chunk):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    g = torch.Generator().manual_seed(0)
    vocab = model.config.vocab_size
    positions = SHORT * (SHORT_PROMPT + SHORT_NEW) + sum(n + LONG_NEW for n in LONG) + 64 * 64
    kw = {"max_prefill_tokens": chunk, "chunked_prefill": True} if chunk else {}
    engine = ContinuousBatcher(model, max_cache_tokens=positions, kv_cache_dtype=dtype, **kw)
    for _ in range(SHORT):
        engine.submit(torch.randint(0, vocab, (SHORT_PROMPT,), generator=g).tolist(), SHORT_NEW)
    longs = [torch.randint(0, vocab, (n,), generator=g).tolist() for n in LONG]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seen, last, gaps, submitted, ttft = {}, {}, [], {}, {}
    steps, generated = 0, 0
    while engine.has_work() or len(submitted) < len(LONG):
        if steps >= LONG_EVERY and steps % LONG_EVERY == 0 and len(submitted) < len(LONG):
            submitted[engine.submit(longs[len(submitted)], LONG_NEW)] = time.perf_counter()
        done = engine.step()
        now = time.perf_counter()
        steps += 1
        counts = {r.rid: len(r.tokens) for r in engine._running}
        counts.update({rid: len(toks) for rid, toks in done})
        for rid, n in counts.items():
            prev = seen.get(rid)
            if prev is None or n > prev:
                generated += n - (n - 1 if prev is None else prev)
                if rid in submitted:
                    ttft.setdefault(rid, now - submitted[rid])
                elif rid in last:
                    gaps.append(now - last[rid])
                last[rid] = now
            seen[rid] = n
    wall = time.perf_counter() - t0
    q = statistics.quantiles(gaps, n=100)
    return {"gap_p50_ms": round(q[49] * 1e3, 2), "gap_p99_ms": round(q[98] * 1e3, 2),
            "gap_max_ms": round(max(gaps) * 1e3, 2),
            "ttft_ms": [round(ttft[r] * 1e3, 1) for r in submitted], "tokens_per_s": round(generated / wall, 1),
            "generated": generated, "steps": steps, "wall_s": round(wall, 2)}


def _median_row(runs):
    """Per-metric median over rounds; the spread of the p99 gap and of tokens/s; every round."""
    med = {k: statistics.median(r[k] for r in runs) for k in runs[0] if k != "ttft_ms"}
    med["ttft_ms"] = [statistics.median(r["ttft_ms"][i] for r in runs) for i in range(len(runs[0]["ttft_ms"]))]
    med["gap_p99_ms_range"] = [min(r["gap_p99_ms"] for r in runs), max(r["gap_p99_ms"] for r in runs)]
    med["tokens_per_s_range"] = [min(r["tokens_per_s"] for r in runs), max(r["tokens_per_s"] for r in runs)]
    med["rounds"] = runs
    return med


def engine_rows(chunk: int, rounds: int):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    rows = []
    for name, cfg in (("bloom-560m", BloomConfig.bloom_560m()), ("bloom-3b", BloomConfig.bloom_3b())):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = BloomForCausalLM(cfg).to(torch.bfloat16).eval()
        run_engine(model, None, chunk)                     # warm-up: modules, allocator, every kernel shape
        arms = [(dtype, c) for dtype in (None, torch.float8_e4m3fn) for c in (0, chunk)]
        runs = {arm: [] for arm in arms}
        for _ in range(rounds):
            for dtype, c in arms:
                runs[(dtype, c)].append(run_engine(model, dtype, c))
                print(json.dumps({"model": name, "pools": "fp8" if dtype is not None else "bf16", "chunk": c,
                                  **runs[(dtype, c)][-1]}), flush=True)
        for dtype, c in arms:
            row = {"model": name, "pools": "fp8" if dtype is not None else "bf16", "chunked_prefill": bool(c),
                   "max_prefill_tokens": c or 8192, **_median_row(runs[(dtype, c)])}
            print(json.dumps({k: v for k, v in row.items() if k != "rounds"}), flush=True)
            rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="chunked_bench.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1024, help="max_prefill_tokens of the chunked engine")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("chunked_bench.py measures on a GPU; none is visible")
    result = {"card": card(), "engine": engine_rows(args.chunk, args.rounds), "card_after": card()}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
