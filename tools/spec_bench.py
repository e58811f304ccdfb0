"""Times speculative decoding: the paged append-attention kernel, the cost of a verify step against a decode step,
and ContinuousBatcher end to end with prompt-lookup drafts.

    python tools/spec_bench.py --out profiles/spec_decode_h100.json [--iters 50] [--requests 256]

Kernel: for B·H in {16, 128, 512} (H = 16), cache length L in {512, 2048, 8192, 32768}, n in {1, 2, 4, 8} appended
tokens per row and D in {64, 128}, every row holds L keys after the call (positions L - n .. L - 1 are the new ones).
One ``alibi_paged_append_attention`` call, one ``alibi_paged_prefill_attention`` call on the same tokens and pools
(the paged prefill kernel, which reads the new keys from the pools), and one ``alibi_paged_decode_attention`` call
(one token per row at position L - 1) are timed with CUDA events over ``--iters`` launches after warm-up.  K+V
bandwidth is the keys and values of the L positions of every (row, head) once, over the time.

Step cost: random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80) with R in {1, 8, 32, 128} running requests of
512 cached positions.  A decode step is ``_paged_logits`` on one token per request plus the arg-max and its transfer
to the host, as the engine runs it; a verify step is ``_paged_logits`` in append mode on the last token and k drafts
per request plus ``verify_drafts`` (greedy), for k in {3, 7}.  Both are timed on the host around work that ends in
the device-to-host transfer, median of ``--step-iters``.  The ratio is the cost of checking k drafts in units of one
decode step, and does not depend on the weights.

End to end: the tools/serve_bench.py workload (256 greedy requests, prompts log-uniform in [16, 1024], max_new_tokens
uniform in [16, 256], seed 0) on random-init bf16 bloom-560m through one ContinuousBatcher per arm with
num_speculative_tokens k in {0, 3, 5, 7}; the arms alternate in this process after a warm-up of each.  The models
are random-init: there is no trained checkpoint, so the acceptance rate (and with it the speed-up) says nothing about
real text.  The workload's prompts are uniform random tokens; a random-init model's greedy continuation often falls
into repetition, which prompt lookup then predicts.

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
from decode_bench import card, time_us  # noqa: E402
from serve_bench import MAX_NEW, MAX_PROMPT, STATIC_BATCH, workload  # noqa: E402


def kernel_rows(iters: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_paged_append_attention, alibi_paged_decode_attention,
                                              alibi_paged_prefill_attention)

    rows = []
    H = 16
    for BH in (16, 128, 512):
        B = BH // H
        for D in (64, 128):
            for length in (512, 2048, 8192, 32768):
                n_pages = length // PAGE_SIZE
                g = torch.Generator(device="cuda").manual_seed(length + D + BH)
                table = torch.randperm(B * n_pages, device="cuda", generator=g).to(torch.int32).view(B, n_pages)
                k_pool = torch.randn(B * n_pages, H, PAGE_SIZE, D, device="cuda", generator=g, dtype=torch.bfloat16)
                v_pool = torch.randn(B * n_pages, H, PAGE_SIZE, D, device="cuda", generator=g, dtype=torch.bfloat16)
                slopes = K.alibi_slopes(H, device="cuda")
                kv_bytes = B * H * length * D * 2 * 2
                qkv1 = torch.randn(B, H * 3 * D, device="cuda", generator=g, dtype=torch.bfloat16)
                last = torch.full((B,), length - 1, dtype=torch.int32, device="cuda")
                t_dec = time_us(lambda: alibi_paged_decode_attention(qkv1, k_pool, v_pool, table, last, length - 1,
                                                                     slopes, D), iters)
                for n in (1, 2, 4, 8):
                    qkv = torch.randn(B * n, H * 3 * D, device="cuda", generator=g, dtype=torch.bfloat16)
                    cu = torch.arange(0, B * n + 1, n, dtype=torch.int32, device="cuda")
                    pos = torch.full((B,), length - n, dtype=torch.int32, device="cuda")
                    t_app = time_us(lambda: alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos,
                                                                         length - 1, slopes, D, max_tokens=n), iters)
                    t_pre = time_us(lambda: alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, pos, n,
                                                                          slopes, D), iters)
                    row = {"B": B, "H": H, "BH": BH, "D": D, "len": length, "n": n,
                           "append_us": round(t_app, 2), "prefill_kernel_us": round(t_pre, 2),
                           "decode_us": round(t_dec, 2), "prefill_over_append": round(t_pre / t_app, 2),
                           "append_over_decode": round(t_app / t_dec, 3), "kv_bytes": kv_bytes,
                           "append_kv_TBps": round(kv_bytes / t_app / 1e6, 3),
                           "prefill_kv_TBps": round(kv_bytes / t_pre / 1e6, 3),
                           "decode_kv_TBps": round(kv_bytes / t_dec / 1e6, 3)}
                    print(json.dumps(row), flush=True)
                    rows.append(row)
                del k_pool, v_pool
                torch.cuda.empty_cache()
    return rows


def _model(name):
    import torch

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    cfg = BloomConfig.bloom_560m() if name == "bloom-560m" else BloomConfig.bloom_3b()
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = BloomForCausalLM(cfg)
    return model.to(torch.bfloat16).eval()


def step_rows(iters: int, context: int = 512):
    import torch

    from pipegoose_b200.ops.attention import PAGE_SIZE
    from pipegoose_b200.serving import verify_drafts

    rows = []
    for name in ("bloom-560m", "bloom-3b"):
        model = _model(name)
        cfg = model.config
        D = cfg.hidden_size // cfg.n_head
        for R in (1, 8, 32, 128):
            pages = (context + 8) // PAGE_SIZE + 1
            shape = (cfg.n_layer, R * pages, cfg.n_head, PAGE_SIZE, D)
            k_pools = torch.randn(shape, device="cuda", dtype=torch.bfloat16)
            v_pools = torch.randn(shape, device="cuda", dtype=torch.bfloat16)
            table = torch.arange(R * pages, dtype=torch.int32, device="cuda").view(R, pages)

            def timed(fn):
                for _ in range(3):
                    fn()
                ts = []
                for _ in range(iters):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    ts.append((time.perf_counter() - t0) * 1e3)
                return statistics.median(ts)

            def decode():
                ids = torch.randint(0, 1000, (R,), dtype=torch.int32).to("cuda")
                pos = torch.full((R,), context, dtype=torch.int32).to("cuda")
                lg = model._paged_logits(ids, pos, k_pools, v_pools, table=table, max_pos=context)
                return lg.float().argmax(-1).tolist()

            row = {"model": name, "D": D, "requests": R, "context": context, "decode_step_ms": round(timed(decode), 3)}
            for k in (3, 7):
                def verify():
                    n = k + 1
                    ids = torch.randint(0, 1000, (R * n,), dtype=torch.int32)
                    pos = (context + torch.arange(n, dtype=torch.int32)).repeat(R)
                    cu = torch.arange(0, R * n + 1, n, dtype=torch.int32)
                    dev = torch.cat([ids, pos, cu]).to("cuda").split([R * n, R * n, R + 1])
                    lg = model._paged_logits(dev[0], dev[1], k_pools, v_pools, table=table, max_pos=context + k,
                                             cu_seqlens=dev[2], max_len=n)
                    drafts = [ids[i * n + 1:(i + 1) * n].tolist() for i in range(R)]
                    return verify_drafts([(False,)] * R, drafts, dev[0], lg.float())

                t = timed(verify)
                row[f"verify_k{k}_ms"] = round(t, 3)
                row[f"verify_k{k}_over_decode"] = round(t / row["decode_step_ms"], 3)
            print(json.dumps(row), flush=True)
            rows.append(row)
            del k_pools, v_pools
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    return rows


def run_engine(model, prompts, news, k):
    import torch

    from pipegoose_b200.serving import ContinuousBatcher

    engine = ContinuousBatcher(model, max_cache_tokens=STATIC_BATCH * (MAX_PROMPT + MAX_NEW), num_speculative_tokens=k)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rids = [engine.submit(p, n) for p, n in zip(prompts, news)]
    finish, steps = {}, 0
    while engine.has_work():
        done = engine.step()
        steps += 1
        now = time.perf_counter()
        for rid, _ in done:
            finish[rid] = now - t0
    return [finish[r] for r in rids], time.perf_counter() - t0, steps, engine


def e2e_rows(n_requests: int, rounds: int):
    prompts, news = workload(n_requests)
    warm_p, warm_n = workload(16, seed=1)
    model = _model("bloom-560m")
    ks = (0, 3, 5, 7)
    for k in ks:
        run_engine(model, warm_p, warm_n, k)
    res = {k: [] for k in ks}
    outs = {}
    for _ in range(rounds):
        for k in ks:
            lat, wall, steps, eng = run_engine(model, prompts, news, k)
            res[k].append((lat, wall, steps, eng.speculative_proposed_tokens, eng.speculative_accepted_tokens))
    rows = []
    for k in ks:
        walls = [r[1] for r in res[k]]
        i = walls.index(statistics.median(walls)) if len(walls) % 2 else walls.index(min(walls))
        lat, wall, steps, proposed, accepted = res[k][i]
        lat = sorted(lat)
        row = {"model": "bloom-560m", "k": k, "requests": n_requests, "generated_tokens": sum(news),
               "tokens_per_s": round(sum(news) / wall, 1), "wall_s": round(wall, 3),
               "p50_latency_s": round(statistics.median(lat), 3),
               "p95_latency_s": round(lat[min(len(lat) - 1, int(0.95 * len(lat)))], 3), "steps": steps,
               "proposed": proposed, "accepted": accepted,
               "acceptance_rate": round(accepted / proposed, 3) if proposed else None,
               "wall_s_samples": [round(w, 3) for w in walls]}
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="spec_bench.json")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--step-iters", type=int, default=20)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernel, step, e2e")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("spec_bench.py measures on a GPU; none is visible")
    skip = set(filter(None, args.skip.split(",")))
    result = {"card": card()}
    if "kernel" not in skip:
        result["kernel"] = kernel_rows(args.iters)
    if "step" not in skip:
        result["step"] = step_rows(args.step_iters)
    if "e2e" not in skip:
        result["e2e"] = e2e_rows(args.requests, args.rounds)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
