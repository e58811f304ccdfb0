"""FP8 against bf16 linear layers on one GPU: per-layer times and training-step times, written to
``profiles/fp8_train_h100.json`` (or ``--out``) with the card's name and power limit read in the same run.

Per layer (qkv, dense, fc1, fc2 of a Bloom block at ``--tokens`` tokens and h in ``--widths``):
  bf16 forward  : GEMM + bias (+ GELU with the pre-activation for fc1)
  bf16 backward : dgrad GEMM, wgrad GEMM into an fp32 main grad with the fused bias gradient
  FP8 forward   : e4m3 casts of the input and the weight (each with its transposed codes) + FP8 GEMM with the same epilogue
  FP8 backward  : e5m2 cast of dY (with transposed codes and the bias column sums) + FP8 dgrad + FP8 wgrad into the main grad
The FP8 times include every cast.  Training steps: bloom-560m at bench.py's configuration (8 x 1024 tokens, FusedAdam)
and bloom-1b7 at the same batch, switching the blocks between the two arms.  Arms alternate after warm-up in one
process; each number is the median over rounds.

    python tools/fp8_train_bench.py                    # everything
    python tools/fp8_train_bench.py --skip-steps       # per-layer table only
    python tools/fp8_train_bench.py --profile-out p.json --widths 1024   # where an FP8 forward's time goes, only

``--profile-out``: for qkv and dense at each width, one FP8 forward (two casts and the GEMM) timed with events over 20
calls, and the same 20 calls under ``torch.profiler``: the device time of each kernel and memset per call, their sum,
and the rest of the event time (the device waiting between kernels).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        idx = torch.cuda.current_device()
        power, clock = [s.strip() for s in q[idx].split(",")]
    except Exception as e:  # the number is still reported; say why the card's limits are missing
        power, clock = f"unknown ({e})", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def layer_arms(M, K_in, N, gelu):
    from pipegoose_b200.ops import kernels as K

    dev = "cuda"
    x = (torch.randn(M, K_in, device=dev)).to(torch.bfloat16)
    w = (torch.randn(N, K_in, device=dev) / K_in ** 0.5).to(torch.bfloat16)
    b = torch.zeros(N, dtype=torch.bfloat16, device=dev)
    dy = (torch.randn(M, N, device=dev) * 1e-3).to(torch.bfloat16)
    z = torch.empty(M, N, dtype=torch.bfloat16, device=dev) if gelu else None
    mg = torch.zeros(N, K_in, dtype=torch.float32, device=dev)
    mgb = torch.zeros(N, dtype=torch.float32, device=dev)

    def bf16_fwd():
        K.gemm_nt(x, w, b, gelu=gelu, aux_out=z)

    def bf16_bwd():
        K.gemm_nn(dy, w)
        K.gemm_tn(dy, x, accum_into=mg, accumulate=True, bias_grad=mgb)

    saved = {}

    def fp8_fwd():
        xc, xt, sx = K.fp8_quantize(x, "e4m3", transpose=True)
        wc, wt, sw = K.fp8_quantize(w, "e4m3", transpose=True)
        K.gemm_fp8(xc, wc, sx, sw, bias=b, gelu=gelu, aux_out=z)
        saved.update(xt=xt, sx=sx, wt=wt, sw=sw)

    def fp8_bwd():
        dc, dt, sd = K.fp8_quantize(dy, "e5m2", transpose=True, colsum_into=mgb)
        K.gemm_fp8(dc, saved["wt"], sd, saved["sw"])
        K.gemm_fp8(dt, saved["xt"], sd, saved["sx"], accum_into=mg, accumulate=True)

    return {"bf16": (bf16_fwd, bf16_bwd), "fp8": (fp8_fwd, fp8_bwd)}


def bench_layers(tokens, widths, rounds, iters):
    out = []
    for h in widths:
        for name, K_in, N, gelu in (("qkv", h, 3 * h, False), ("dense", h, h, False), ("fc1", h, 4 * h, True),
                                    ("fc2", 4 * h, h, False)):
            arms = layer_arms(tokens, K_in, N, gelu)
            for fwd, bwd in arms.values():  # warm-up (module load, tensor maps)
                fwd(), bwd()
                time_ms(fwd, iters), time_ms(bwd, iters)
            t = {a: {"fwd": [], "bwd": []} for a in arms}
            for _ in range(rounds):
                for a, (fwd, bwd) in arms.items():
                    t[a]["fwd"].append(time_ms(fwd, iters))
                    t[a]["bwd"].append(time_ms(bwd, iters))
            row = {"h": h, "layer": name, "M": tokens, "K": K_in, "N": N}
            for a in arms:
                for d in ("fwd", "bwd"):
                    row[f"{a}_{d}_us"] = round(1e3 * statistics.median(t[a][d]), 1)
            row["speedup_fwd_bwd"] = round((row["bf16_fwd_us"] + row["bf16_bwd_us"]) /
                                           (row["fp8_fwd_us"] + row["fp8_bwd_us"]), 3)
            print(json.dumps(row), flush=True)
            out.append(row)
            del arms
            torch.cuda.empty_cache()
    return out


def profile_fp8_fwd(tokens, widths, iters=20):
    from torch.profiler import ProfilerActivity, profile

    out = []
    for h in widths:
        for name, K_in, N in (("qkv", h, 3 * h), ("dense", h, h)):
            fwd = layer_arms(tokens, K_in, N, False)["fp8"][0]
            for _ in range(5):
                fwd()
            time_ms(fwd, iters)
            event_us = 1e3 * statistics.median(time_ms(fwd, iters) for _ in range(5))
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    fwd()
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                if t > 0:
                    kernels[e.key] = round(t / iters, 2)
            busy = sum(kernels.values())
            row = {"h": h, "layer": name, "M": tokens, "K": K_in, "N": N, "event_us": round(event_us, 1),
                   "device_busy_us": round(busy, 1), "device_idle_us": round(event_us - busy, 1),
                   "kernels_us": dict(sorted(kernels.items(), key=lambda kv: -kv[1]))}
            print(json.dumps(row), flush=True)
            out.append(row)
    return out


def bench_steps(model_name, batch, seq, warmup, steps, rounds):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.optim import FusedAdam

    torch.manual_seed(0)
    cfg = getattr(BloomConfig, model_name.replace("-", "_"))()
    model = BloomForCausalLM(cfg).to(torch.bfloat16).cuda()
    opt = FusedAdam(model.parameters(), lr=1e-4)
    ids = torch.randint(0, cfg.vocab_size, (batch, seq), device="cuda")

    def set_arm(fp8):
        for blk in model.transformer.h:
            blk.fp8 = fp8

    def run(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            loss = model(ids, labels=ids).loss
            opt.zero_grad()
            loss.backward()
            opt.step()
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / n, loss.item()

    for fp8 in (False, True):
        set_arm(fp8)
        run(warmup)
    t = {"bf16": [], "fp8": []}
    loss = {}
    for _ in range(rounds):
        for arm in ("bf16", "fp8"):
            set_arm(arm == "fp8")
            ms, loss[arm] = run(steps)
            t[arm].append(ms)
    row = {"model": model_name, "batch": batch, "seq_len": seq, "optimizer": "FusedAdam",
           "bf16_ms": [round(v, 2) for v in t["bf16"]], "fp8_ms": [round(v, 2) for v in t["fp8"]],
           "bf16_median_ms": round(statistics.median(t["bf16"]), 2),
           "fp8_median_ms": round(statistics.median(t["fp8"]), 2),
           "last_loss": {k: round(v, 4) for k, v in loss.items()},
           "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)}
    row["speedup"] = round(row["bf16_median_ms"] / row["fp8_median_ms"], 3)
    print(json.dumps(row), flush=True)
    del model, opt
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "fp8_train_h100.json"))
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--widths", default="1024,2560,4096")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--step-models", default="bloom-560m,bloom-1b7")
    ap.add_argument("--profile-out", default="", help="write only the FP8 forward profile, to this file")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seq-len", type=int, default=1024)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_train_bench needs a GPU")
    from pipegoose_b200 import ops

    ops.native()
    if args.profile_out:
        res = {"card": card(), "tokens": args.tokens,
               "fp8_forward_profile": profile_fp8_fwd(args.tokens, [int(w) for w in args.widths.split(",")])}
        with open(args.profile_out, "w") as f:
            json.dump(res, f, indent=1)
        print(f"wrote {args.profile_out}")
        return
    res = {"card": card(), "tokens": args.tokens,
           "layers": bench_layers(args.tokens, [int(w) for w in args.widths.split(",")], args.rounds, args.iters)}
    if not args.skip_steps:
        res["steps"] = [bench_steps(m, args.batch, args.seq_len, 3, 5, args.rounds) for m in args.step_models.split(",")]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
