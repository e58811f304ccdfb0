"""Where the flash-attention backward's time goes, launch by launch, and what attention costs in a training step.

    python tools/attn_bwd_bench.py --out /tmp/attn_bwd.json                       # the extension in the tree
    python tools/attn_bwd_bench.py --exts ,parent --rounds 3 --out ...            # alternate _C.so and _C_parent.so
    python tools/attn_bwd_bench.py --step-profile --out ...                       # + kernel table of one bench step

For each extension (``""`` is ``pipegoose_b200/_C.so``, a name loads the variant build ``_C_<name>.so``) and each shape:
  * ``call_us``: one ``attention_bwd`` call (every launch it makes), CUDA events around 50 calls;
  * ``launches``: the device time of each kernel / memset of the call, from ``torch.profiler`` (CUDA activities) over
    20 calls in a separate, traced window;
  * ``fwd_us``: the forward at the same shape, for scale.
Every extension runs in its own process, rounds alternate between them.  ``--step-profile`` traces one bloom-560m
training step (8 x 1024 tokens, forward, backward, Adam) after warm-up and prints its kernels by total device time.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(8, 1024, 16, 64), (4, 2048, 32, 128)]  # bloom-560m; bloom-3b/7b1-sized heads


def _kernel_times(prof, n_calls):
    """{name: (launches per call, device us per call)} of the CUDA activities in a profiler window."""
    import torch

    out = {}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        # template instantiations of one kernel share the name: add them up
        name = e.key.split("(")[0].split("<")[0].strip()
        c0, us0 = out.get(name, (0.0, 0.0))
        out[name] = (c0 + e.count / n_calls, us0 + us / n_calls)
    return out


def _time_us(fn, iters):
    import torch

    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def worker():
    import torch
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, ROOT)
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops import native

    n = native()
    torch.manual_seed(0)
    res = []
    for B, S, H, D in SHAPES:
        qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
        slopes = K.alibi_slopes(H, device="cuda")
        out = torch.empty(B * S, H * D, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(B, H, S, device="cuda")
        dout = torch.randn_like(out)
        dqkv = torch.empty_like(qkv)
        fwd = lambda: n.attention_fwd(qkv, slopes, out, lse, B, S, H, D)  # noqa: E731
        bwd = lambda: n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D)  # noqa: E731
        fwd()
        for _ in range(5):
            bwd()
        fwd_us = _time_us(fwd, 50)
        call_us = _time_us(bwd, 50)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                bwd()
            torch.cuda.synchronize()
        launches = {k: {"per_call": round(c, 2), "us": round(us, 1)} for k, (c, us) in _kernel_times(prof, 20).items()}
        flop = 4 * B * H * S * S * D / 2 * 2.5  # causal half, backward charged 2.5 x the forward
        res.append({"B": B, "S": S, "H": H, "D": D, "fwd_us": round(fwd_us, 1), "call_us": round(call_us, 1),
                    "bwd_tflops": round(flop / call_us / 1e6, 1), "launches": launches})
        del qkv, out, lse, dout, dqkv
    return res


def step_profile():
    import torch
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, ROOT)
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.optim.fused_adam import FusedAdam

    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    cfg = BloomConfig.bloom_560m()
    model = BloomForCausalLM(cfg).to(torch.bfloat16).to(dev)
    optim = FusedAdam(model.parameters(), lr=1e-4)
    ids = torch.randint(0, cfg.vocab_size, (8, 1024), device=dev)

    def step():
        loss = model(ids, labels=ids).loss
        optim.zero_grad()
        loss.backward()
        optim.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kt = _kernel_times(prof, 1)
    total = sum(us for _, us in kt.values())
    table = sorted(({"name": k, "count": int(c), "us": round(us, 1), "frac": round(us / total, 4)} for k, (c, us) in kt.items()),
                   key=lambda r: -r["us"])
    att = sum(r["us"] for r in table if "attention" in r["name"] or r["name"].startswith("Memset"))
    return {"kernel_us": round(total, 1), "attention_us": round(att, 1), "kernels": table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--exts", default="", help="comma-separated extension variants; '' is the main _C.so")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--step-profile", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker is not None:
        print(json.dumps(step_profile() if args.worker == "step" else worker()))
        return
    exts = args.exts.split(",")
    runs = []
    for r in range(args.rounds):
        for ext in exts:
            env = dict(os.environ, PIPEGOOSE_B200_EXT=ext)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "shapes"], env=env,
                               capture_output=True, text=True, check=True)
            res = json.loads(p.stdout.strip().splitlines()[-1])
            runs.append({"round": r, "ext": ext or "main", "shapes": res})
            for s in res:
                split = "  ".join(f"{k} {v['us']:.1f}" for k, v in sorted(s["launches"].items(), key=lambda kv: -kv[1]["us"]))
                print(f"round {r} {ext or 'main':>10}  {s['B']}x{s['S']}x{s['H']}x{s['D']}  fwd {s['fwd_us']:7.1f} us  "
                      f"bwd call {s['call_us']:7.1f} us ({s['bwd_tflops']} TFLOP/s)  | {split}", flush=True)
    out = {"runs": runs}
    if args.step_profile:
        for ext in exts:
            env = dict(os.environ, PIPEGOOSE_B200_EXT=ext)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "step"], env=env,
                               capture_output=True, text=True, check=True)
            sp = json.loads(p.stdout.strip().splitlines()[-1])
            out.setdefault("step_profile", {})[ext or "main"] = sp
            print(f"step profile {ext or 'main'}: {sp['kernel_us'] / 1e3:.2f} ms of kernels, attention "
                  f"{sp['attention_us'] / 1e3:.2f} ms")
            for k in sp["kernels"][:30]:
                print(f"  {k['us']:9.1f} us {k['frac'] * 100:5.1f}% x{k['count']:<4d} {k['name'][:90]}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
