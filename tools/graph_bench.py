"""Times ContinuousBatcher's decode step eager and replayed from CUDA graphs (``cuda_graphs=True``).

    python tools/graph_bench.py --out profiles/cuda_graphs_h100.json [--rounds 6] [--e2e-rounds 2] [--skip-e2e]

Decode step: random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80), B in {1, 8, 64, 256} greedy requests with
prompts of ``PROMPT`` tokens, prefilled first.  The step is one ``engine.step()``, which ends in the device-to-host
transfer of the chosen tokens, timed with CUDA events around it.  One engine serves both arms (its ``cuda_graphs``
switched off for the eager arm, so both arms decode the same requests over the same pools), alternating ``--steps``
steps of each arm for ``--rounds`` rounds after a warm-up step of each; the context grows by one position per step,
from ``PROMPT`` to at most ``PROMPT + 2 + 2 * rounds * steps`` positions.  Reported: the median step time of each arm
with its min and max, and the memory the capture of the bucket adds (``torch.cuda.memory_stats`` around it, the
allocator's cache emptied first: the graph pool, the static logits and, on the engine's first capture, cuBLAS's
workspace for the capture stream), with the capture's wall time.

End to end: the workload of tools/serve_bench.py (256 requests, prompts log-uniform in [16, 1024], max_new_tokens
uniform in [16, 256], one engine with a pool of 32 x 1280 positions), with ``cuda_graphs`` off and on, alternating
``--e2e-rounds`` rounds after a warm-up of each arm on 16 requests; each arm reports the round with the median wall time
(with an even number of rounds, the fastest) and all wall times.

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
from serve_bench import MAX_NEW, MAX_PROMPT, STATIC_BATCH, workload  # noqa: E402

PROMPT = 512
BATCHES = (1, 8, 64, 256)
MODELS = ("bloom-560m", "bloom-3b")


def _model(name):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    cfg = BloomConfig.bloom_560m() if name == "bloom-560m" else BloomConfig.bloom_3b()
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = BloomForCausalLM(cfg)
    return model.to(torch.bfloat16).eval()


def _timed_step(engine, graphs: bool) -> float:
    import torch

    engine.cuda_graphs = graphs
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    engine.step()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3


def decode_rows(rounds: int, steps: int):
    import torch

    from pipegoose_b200.ops.attention import PAGE_SIZE
    from pipegoose_b200.serving import ContinuousBatcher

    rows = []
    new = 4 + 2 * rounds * steps                       # no request finishes inside the timed steps
    for name in MODELS:
        model = _model(name)
        for B in BATCHES:
            pages = -(-(PROMPT + new) // PAGE_SIZE)
            engine = ContinuousBatcher(model, max_cache_tokens=B * pages * PAGE_SIZE, cuda_graphs=True)
            g = torch.Generator().manual_seed(B)
            for _ in range(B):
                engine.submit(torch.randint(0, model.config.vocab_size, (PROMPT,), generator=g).tolist(), new)
            while engine._admitted or engine._waiting:
                engine.step()                                  # prefill
            assert len(engine._running) == B
            n = next(s for s in engine._graph_sizes if s >= B)
            torch.cuda.synchronize()
            torch.cuda.empty_cache()                          # capture empties the cache: compare like with like
            before = torch.cuda.memory_stats()
            t0 = time.perf_counter()
            engine._graph(n)
            torch.cuda.synchronize()
            capture_s = time.perf_counter() - t0
            after = torch.cuda.memory_stats()
            _timed_step(engine, False)
            _timed_step(engine, True)
            times = {"eager": [], "graph": []}
            for _ in range(rounds):
                for arm in ("eager", "graph"):
                    times[arm] += [_timed_step(engine, arm == "graph") for _ in range(steps)]
            assert len(engine._running) == B and engine.graph_decode_steps == 1 + rounds * steps
            row = {"model": name, "B": B, "bucket": n, "context_positions": [PROMPT, PROMPT + 2 + 2 * rounds * steps],
                   "table_width_pages": engine._graph_width}
            for arm, t in times.items():
                row[f"{arm}_step_us"] = {"median": round(statistics.median(t), 1), "min": round(min(t), 1),
                                         "max": round(max(t), 1), "n": len(t)}
            row["graph_over_eager"] = round(row["graph_step_us"]["median"] / row["eager_step_us"]["median"], 3)
            row["capture_s"] = round(capture_s, 3)
            for key in ("reserved_bytes.all.current", "allocated_bytes.all.current"):
                row[f"capture_delta_{key.split('.')[0]}_MiB"] = round((after[key] - before[key]) / 2 ** 20, 1)
            print(json.dumps(row), flush=True)
            rows.append(row)
            del engine
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    return rows


def run_engine(model, prompts, news, graphs: bool):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=STATIC_BATCH * (MAX_PROMPT + MAX_NEW), cuda_graphs=graphs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for p, n in zip(prompts, news):
        engine.submit(p, n)
    steps = 0
    while engine.has_work():
        engine.step()
        steps += 1
    wall = time.perf_counter() - t0
    return wall, steps, engine.graph_decode_steps


def e2e_rows(rounds: int):
    import torch

    prompts, news = workload(256)
    warm_p, warm_n = workload(16, seed=1)
    rows = []
    for name in MODELS:
        model = _model(name)
        for graphs in (False, True):
            run_engine(model, warm_p, warm_n, graphs)
        runs = {False: [], True: []}
        for _ in range(rounds):
            for graphs in (False, True):
                runs[graphs].append(run_engine(model, prompts, news, graphs))
        row = {"model": name, "requests": len(prompts), "generated_tokens": sum(news),
               "prompt_tokens": sum(len(p) for p in prompts),
               "engine_pool_positions": STATIC_BATCH * (MAX_PROMPT + MAX_NEW)}
        for graphs, res in runs.items():
            walls = [w for w, _, _ in res]
            i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
            row["graphs" if graphs else "eager"] = {
                "tokens_per_s": round(sum(news) / walls[i], 1), "wall_s": round(walls[i], 3), "steps": res[i][1],
                "graph_decode_steps": res[i][2], "wall_s_samples": [round(w, 3) for w in walls]}
        row["graphs_over_eager_tokens_per_s"] = round(row["graphs"]["tokens_per_s"] / row["eager"]["tokens_per_s"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="graph_bench.json")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=5, help="decode steps of one arm per round")
    ap.add_argument("--e2e-rounds", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("graph_bench.py measures on a GPU; none is visible")
    result = {"card": card(), "decode_step": decode_rows(args.rounds, args.steps)}
    if not args.skip_e2e:
        result["e2e"] = e2e_rows(args.e2e_rounds)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
