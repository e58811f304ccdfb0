"""Times KV-cached decoding: the split-KV decode-attention kernel, and generate() with the native path against eager.

    python tools/decode_bench.py --out decode.json [--iters 50] [--skip-e2e]

Kernel: for B·H in {16, 128, 512} (H = 16), filled length in {512, 2048, 8192, 32768} and D in {64, 128}, with and
without left pads (``lead[b]`` spread over the first quarter of the cache), one ``alibi_decode_attention`` call is timed
with CUDA events over ``--iters`` launches after warm-up, and so is the eager path's formula on the same tensors
(``cat`` onto the cache, fp32 scores, ALiBi, masks, softmax, bf16 ``matmul`` with V).  The bandwidth counts the bytes the
kernel has to move: one bf16 read of every visible key and value, ``2·B·H·len·D·2``, plus the qkv row, the output and
the cache write; it is reported against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).

End to end: ``generate()`` of a random-init bf16 bloom-560m (D = 64) and bloom-3b (D = 80), B in {1, 8}, prompts of 128
and 2048 tokens, 128 greedy new tokens.  The native arm and the eager arm alternate in this process; the eager arm is
selected by replacing ``models.bloom._native_decode``, the dispatch predicate, here.  ms/token is
``(t(128 new) - t(1 new)) / 127``; the prefill time is ``t(1 new)``; the peak memory is the rise of
``torch.cuda.max_memory_allocated`` over a 1-token generate (the prompt's working set).

The card name and power limit are read in the same run and written next to the numbers."""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    first = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [p.strip() for p in first.split(",")] if first else []
    return {"gpu": parts[0] if parts else None, "power_limit": parts[1] if len(parts) > 1 else None,
            "max_sm_clock": parts[2] if len(parts) > 2 else None}


def kernel_bytes(B, H, D, pos, lead) -> int:
    """Bytes the decode step has to move: visible keys and values once, the qkv rows, the output and the new k / v."""
    keys = sum(pos + 1 - min(l, pos) for l in lead) if lead is not None else B * (pos + 1)
    return 2 * H * keys * D * 2 + B * H * 3 * D * 2 + B * H * D * 2 + 2 * B * H * D * 2


def eager_step(qkv, k_cache, v_cache, slopes, pos, lead, D):
    """models/bloom.py's eager attention for one new token, on a cache of ``pos`` filled positions."""
    import torch

    B, H = k_cache.shape[:2]
    x = qkv.view(B, 1, H, 3, D)
    q, k, v = (x[:, :, :, i].transpose(1, 2) for i in range(3))
    k = torch.cat([k_cache[:, :, :pos], k], dim=2)
    v = torch.cat([v_cache[:, :, :pos], v], dim=2)
    S = k.shape[2]
    scores = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(D)
    key_pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
    scores = scores + slopes.view(1, H, 1, 1) * key_pos
    query_pos = torch.arange(pos, pos + 1, device=qkv.device).view(1, 1)
    scores = scores.masked_fill(key_pos.view(1, S) > query_pos, float("-inf"))
    if lead is not None:
        pad = key_pos.view(1, 1, 1, -1) < lead.view(-1, 1, 1, 1).to(key_pos.dtype)
        scores = scores.masked_fill(pad, torch.finfo(scores.dtype).min)
    return torch.matmul(scores.softmax(-1).to(v.dtype), v).transpose(1, 2).reshape(B, H * D)


def time_us(fn, iters: int) -> float:
    import torch

    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters


def kernel_rows(iters: int):
    import torch

    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_decode_attention

    rows = []
    H = 16
    for BH in (16, 128, 512):
        B = BH // H
        for D in (64, 128):
            for length in (512, 2048, 8192, 32768):
                pos = length - 1
                g = torch.Generator(device="cuda").manual_seed(length + D + BH)
                k_cache = torch.randn(B, H, length, D, device="cuda", generator=g, dtype=torch.bfloat16)
                v_cache = torch.randn(B, H, length, D, device="cuda", generator=g, dtype=torch.bfloat16)
                qkv = torch.randn(B, H * 3 * D, device="cuda", generator=g, dtype=torch.bfloat16)
                slopes = K.alibi_slopes(H, device="cuda")
                for padded in (False, True):
                    lead_l = [(b * length) // (4 * B) for b in range(B)] if padded else None
                    lead = None if lead_l is None else torch.tensor(lead_l, device="cuda", dtype=torch.int32)
                    native = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, lead, D)
                    eager = eager_step(qkv, k_cache, v_cache, slopes, pos, lead, D)
                    err = ((native.float() - eager.float()).abs().max() / eager.float().abs().max()).item()
                    t_nat = time_us(lambda: alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, lead, D), iters)
                    t_eag = time_us(lambda: eager_step(qkv, k_cache, v_cache, slopes, pos, lead, D),
                                    max(3, iters // 5))
                    nbytes = kernel_bytes(B, H, D, pos, lead_l)
                    row = {"B": B, "H": H, "BH": BH, "D": D, "len": length, "lead": padded,
                           "native_us": round(t_nat, 2), "eager_us": round(t_eag, 2),
                           "speedup": round(t_eag / t_nat, 2), "bytes": nbytes,
                           "native_TBps": round(nbytes / t_nat / 1e6, 3),
                           "share_of_3.35TBps": round(nbytes / t_nat / 1e6 / (HBM_BYTES_PER_S / 1e12), 3),
                           "rel_err_vs_eager": round(err, 5)}
                    print(json.dumps(row), flush=True)
                    rows.append(row)
                del k_cache, v_cache
                torch.cuda.empty_cache()
    return rows


def e2e_rows(rounds: int):
    import time

    import torch

    from pipegoose_b200.models import bloom
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    native_pred = bloom._native_decode
    rows = []
    for name, cfg in (("bloom-560m", BloomConfig.bloom_560m()), ("bloom-3b", BloomConfig.bloom_3b())):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = BloomForCausalLM(cfg)
        model = model.to(torch.bfloat16).eval()
        for B in (1, 8):
            for P in (128, 2048):
                ids = torch.randint(0, cfg.vocab_size, (B, P), device="cuda")
                res = {"native": {"ms_per_token": [], "prefill_ms": [], "peak_mib": []},
                       "eager": {"ms_per_token": [], "prefill_ms": [], "peak_mib": []}}
                tokens = {}
                for r in range(rounds + 1):          # round 0 warms both arms up
                    for arm in ("native", "eager"):
                        bloom._native_decode = native_pred if arm == "native" else (lambda *a: False)
                        torch.cuda.synchronize()
                        base = torch.cuda.memory_allocated()
                        torch.cuda.reset_peak_memory_stats()
                        t0 = time.perf_counter()
                        model.generate(ids, max_new_tokens=1)
                        torch.cuda.synchronize()
                        t1 = time.perf_counter()
                        peak = torch.cuda.max_memory_allocated() - base
                        out = model.generate(ids, max_new_tokens=128)
                        torch.cuda.synchronize()
                        t2 = time.perf_counter()
                        tokens[arm] = out
                        if r > 0:
                            res[arm]["prefill_ms"].append((t1 - t0) * 1e3)
                            res[arm]["ms_per_token"].append(((t2 - t1) - (t1 - t0)) * 1e3 / 127)
                            res[arm]["peak_mib"].append(peak / 2**20)
                bloom._native_decode = native_pred
                new = tokens["native"][:, P:]
                same = (new == tokens["eager"][:, P:]).float().mean().item()
                row = {"model": name, "B": B, "prompt": P, "new_tokens": 128}
                for arm in ("native", "eager"):
                    row[arm] = {k: round(statistics.median(v), 3) for k, v in res[arm].items()}
                    row[arm]["samples_ms_per_token"] = [round(v, 3) for v in res[arm]["ms_per_token"]]
                row["speedup_per_token"] = round(row["eager"]["ms_per_token"] / row["native"]["ms_per_token"], 3)
                row["same_tokens_fraction"] = round(same, 4)
                print(json.dumps(row), flush=True)
                rows.append(row)
        del model
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="decode_bench.json")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("decode_bench.py measures on a GPU; none is visible")
    result = {"card": card(), "kernel": kernel_rows(args.iters)}
    if not args.skip_e2e:
        result["generate"] = e2e_rows(args.rounds)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
