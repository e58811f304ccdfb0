"""Times beam search in ContinuousBatcher: the fused candidate-choice kernel, the fork copy kernel and the engine.

    python tools/beam_bench.py --out profiles/beam_search_h100.json [--iters 50] [--requests 32]

Kernel: ``beam_topk`` against the PyTorch path it replaces (``.float()``, ``log_softmax``, the add of the beam scores
and ``topk(2W)`` over ``[R, W * V]``), on random bf16 logits of R requests with W beams each, V in {250880, 50257},
W in {2, 4, 8}, R in {1, 8, 32}.  The two arms alternate, ``--iters`` calls each per round over 5 rounds, timed with
CUDA events; reported: the median per-call time of each arm and the bandwidth of one read of the bf16 logits.

``paged_kv_copy``: the pools of bloom-560m (24 layers, 16 heads, D = 64, bf16), 32 and 256 pairs of half pages;
reported: the time per launch and the bytes read and written over it.

End to end: random-init bf16 bloom-560m on the first ``--requests`` requests of tools/serve_bench.py's workload with
``num_beams=4``, in the default engine and with ``cuda_graphs``, against 🤗 ``generate(num_beams=4)`` in bf16 on
``to_hf()`` of the same weights in static batches of 8 prompts.  Arms alternate over ``--e2e-rounds`` rounds after a
warm-up; reported per arm: generated tokens / s (tokens of the best hypotheses; without an eos, each request's
``max_new_tokens``), the median wall time (with an even number of rounds, the fastest), steps and
``beam_page_copies``.  One more run of the default engine with a device synchronise around every step and around
every beam step gives the beam step's share of step time (that run is not one of the timed ones).

The card name and power limit are read in the same run and written next to the numbers."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decode_bench import card  # noqa: E402
from serve_bench import MAX_NEW, MAX_PROMPT, workload  # noqa: E402

BEAMS = 4


def _events_ms(fn, iters):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def kernel_rows(iters):
    import torch

    from pipegoose_b200.ops.kernels import beam_topk

    rows = []
    for V in (250880, 50257):
        for W in (2, 4, 8):
            for R in (1, 8, 32):
                N = R * W
                logits = torch.randn(N, V, device="cuda").to(torch.bfloat16)
                scores = torch.randn(N, device="cuda")
                cu = list(range(0, N + 1, W))

                def fused():
                    return beam_topk(logits, scores, cu, 2 * W)

                def torch_path():
                    lp = torch.log_softmax(logits.float(), -1) + scores.view(-1, 1)
                    return torch.topk(lp.view(R, W * V), 2 * W)

                s, _, _, _ = fused()
                diff = (s - torch_path().values).abs().max().item()      # the same scores, up to fp32 rounding
                arms = {"beam_topk": [], "torch": []}
                for _ in range(5):
                    for name, fn in (("beam_topk", fused), ("torch", torch_path)):
                        fn()
                        arms[name].append(_events_ms(fn, iters))
                ms = {k: statistics.median(v) for k, v in arms.items()}
                gbs = N * V * 2 / (ms["beam_topk"] * 1e-3) / 1e9
                rows.append({"V": V, "W": W, "R": R, "rows": N, "beam_topk_us": ms["beam_topk"] * 1e3,
                             "torch_us": ms["torch"] * 1e3, "speedup": ms["torch"] / ms["beam_topk"],
                             "beam_topk_logit_read_GBps": gbs, "max_score_diff_vs_torch": diff,
                             "spread_us": {k: [min(v) * 1e3, max(v) * 1e3] for k, v in arms.items()}})
                print(json.dumps(rows[-1]), flush=True)
    return rows


def copy_rows(iters):
    import torch

    from pipegoose_b200.ops.attention import paged_kv_copy

    L, pages, H, D = 24, 640, 16, 64
    k = torch.randn(L, pages, H, 64, D, device="cuda").to(torch.bfloat16)
    v = torch.randn_like(k)
    rows = []
    for n in (32, 256):
        pairs = torch.tensor([(i, pages // 2 + i, 32) for i in range(n)], dtype=torch.int32, device="cuda")
        paged_kv_copy(pairs, k, v)
        ms = statistics.median(_events_ms(lambda: paged_kv_copy(pairs, k, v), iters) for _ in range(5))
        moved = 2 * 2 * n * L * H * 32 * D * 2                      # K and V, read and written
        rows.append({"pairs": n, "slots_per_pair": 32, "us": ms * 1e3, "bytes": moved,
                     "GBps": moved / (ms * 1e-3) / 1e9})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def _model():
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(0)
    with torch.device("cuda"):
        model = BloomForCausalLM(BloomConfig.bloom_560m())
    return model.to(torch.bfloat16).eval()


def _engine_run(model, prompts, news, graphs, instrument=False):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=32 * (MAX_PROMPT + MAX_NEW), cuda_graphs=graphs)
    times = {"step": 0.0, "beam": 0.0}
    if instrument:
        step, beam = engine.step, engine._beam_step

        def timed(fn, key):
            def run(*a):
                torch.cuda.synchronize()
                t = time.perf_counter()
                out = fn(*a)
                torch.cuda.synchronize()
                times[key] += time.perf_counter() - t
                return out
            return run
        engine.step, engine._beam_step = timed(step, "step"), timed(beam, "beam")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for p, n in zip(prompts, news):
        engine.submit(p, n, num_beams=BEAMS)
    steps = 0
    outs = {}
    while engine.has_work():
        outs.update(engine.step())
        steps += 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    tokens = sum(len(o) for o in outs.values()) - sum(len(p) for p in prompts)
    res = {"wall_s": wall, "tokens": tokens, "steps": steps, "beam_page_copies": engine.beam_page_copies}
    if instrument:
        res["beam_step_share"] = times["beam"] / times["step"]
    return res


def _hf_run(hf, prompts, news, batch=8):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tokens = 0
    for i in range(0, len(prompts), batch):
        ps, n = prompts[i:i + batch], max(news[i:i + batch])
        width = max(len(p) for p in ps)
        ids = torch.tensor([[0] * (width - len(p)) + p for p in ps], device="cuda")
        mask = torch.tensor([[0] * (width - len(p)) + [1] * len(p) for p in ps], device="cuda")
        out = hf.generate(ids, attention_mask=mask, max_new_tokens=n, num_beams=BEAMS, do_sample=False,
                          eos_token_id=10 ** 6, pad_token_id=0)
        tokens += out.numel() - ids.numel()
    torch.cuda.synchronize()
    # without an eos every best hypothesis runs to its request's max_new_tokens, as in the engine; the batch's longer
    # requests make the others generate more (tokens_generated), but only the requested tokens count
    return {"wall_s": time.perf_counter() - t0, "tokens": sum(news), "tokens_generated": tokens}


def e2e_rows(n_requests, rounds):
    import torch

    model = _model()
    hf = model.to_hf().to(torch.bfloat16).cuda().eval()
    prompts, news = workload(n_requests)
    wp, wn = workload(4, seed=1)
    arms = {"engine": lambda: _engine_run(model, prompts, news, False),
            "engine_cuda_graphs": lambda: _engine_run(model, prompts, news, True),
            "hf_generate": lambda: _hf_run(hf, prompts, news)}
    warm = {"engine": lambda: _engine_run(model, wp, wn, False), "engine_cuda_graphs": lambda: _engine_run(
        model, wp, wn, True), "hf_generate": lambda: _hf_run(hf, wp, wn)}
    for fn in warm.values():
        fn()
    runs = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            runs[k].append(fn())
            print(k, json.dumps(runs[k][-1]), flush=True)
    out = {}
    for k, rs in runs.items():
        best = sorted(rs, key=lambda r: r["wall_s"])[(len(rs) - 1) // 2]
        out[k] = dict(best, tokens_per_s=best["tokens"] / best["wall_s"], wall_s_all=[r["wall_s"] for r in rs])
    out["engine_instrumented"] = _engine_run(model, prompts[:16], news[:16], False, instrument=True)
    print(json.dumps(out["engine_instrumented"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--e2e-rounds", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a GPU")
    res = {"card": card(), "torch": torch.__version__, "kernel": kernel_rows(args.iters),
           "paged_kv_copy": copy_rows(args.iters)}
    if not args.skip_e2e:
        res["e2e"] = dict(e2e_rows(args.requests, args.e2e_rounds), requests=args.requests, num_beams=BEAMS)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
