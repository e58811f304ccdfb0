"""Times the document-masked (packed-sequence) flash attention against the plain causal kernels.

    python tools/packed_attn_bench.py --out packed_attn.json [--ab parent] [--rounds 3]

Per shape (B·S·H·D = 8·1024·16·64, bloom-560m's attention, and 4·2048·32·128) and layout:

* ``unpacked``: ``seg_start=None``, the plain causal kernels;
* ``one_doc``: one document per row through the ``seg_start`` kernels (the cost of the flag itself);
* ``docs256``: 256-token documents;
* ``mix``: a seeded log-uniform mix of document lengths in [32, S], different in every row.

the forward and the backward (delta + main kernel + dQ conversion) are timed with CUDA events over ``--iters`` launches
after warm-up.  "Useful" TFLOP/s count, per document of ``n`` tokens, the causal visible half ``2 n^2 D`` per head for
the forward and 2.5 times that for the backward.  ``--ab NAME`` also times the ``unpacked`` rows with the extension
build ``pipegoose_b200/_C_NAME.so`` (``PIPEGOOSE_B200_BUILD_VARIANT=NAME`` when it was built), alternating the two
builds over ``--rounds`` rounds, each in a fresh process.  Finally one bloom-560m training step (B = 8, S = 1024) is
timed without and with 256-token ``position_ids``.

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
SHAPES = [(8, 1024, 16, 64), (4, 2048, 32, 128)]
LAYOUTS = ["unpacked", "one_doc", "docs256", "mix"]


def doc_lengths(layout: str, B: int, S: int, seed: int = 0):
    """Document lengths of every row (None: unpacked)."""
    import numpy as np

    if layout == "unpacked":
        return None
    if layout == "one_doc":
        return [[S] for _ in range(B)]
    if layout == "docs256":
        return [[256] * (S // 256) + ([S % 256] if S % 256 else []) for _ in range(B)]
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(B):
        row, left = [], S
        while left > 0:
            n = int(round(math.exp(rng.uniform(math.log(32), math.log(S)))))
            n = min(max(n, 32), left)
            row.append(n)
            left -= n
        rows.append(row)
    return rows


def useful_fwd_flops(lengths, B: int, S: int, H: int, D: int) -> float:
    rows = lengths if lengths is not None else [[S]] * B
    return sum(2.0 * n * n * D * H for row in rows for n in row)


def _time(fn, iters: int) -> float:
    import torch

    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3   # µs


def worker_kernels(layouts, iters: int):
    import torch

    sys.path.insert(0, ROOT)
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops import native

    n = native()
    rows = []
    for (B, S, H, D) in SHAPES:
        torch.manual_seed(0)
        qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
        slopes = K.alibi_slopes(H, device="cuda")
        out = torch.empty(B * S, H * D, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(B, H, S, device="cuda")
        dout = torch.randn_like(out)
        dqkv = torch.empty_like(qkv)
        for layout in layouts:
            lengths = doc_lengths(layout, B, S)
            if lengths is None:
                fwd = lambda: n.attention_fwd(qkv, slopes, out, lse, B, S, H, D)                       # noqa: E731
                bwd = lambda: n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D)           # noqa: E731
            else:
                seg = torch.cat([torch.cat([torch.full((m,), s0, dtype=torch.int32)
                                            for s0, m in zip([sum(r[:i]) for i in range(len(r))], r)]) for r in lengths])
                seg = seg.cuda()
                fwd = lambda: n.attention_fwd(qkv, slopes, out, lse, B, S, H, D, 0.0, seg)             # noqa: E731
                bwd = lambda: n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D, 0.0, seg)  # noqa: E731
            fwd_us = _time(fwd, iters)
            bwd_us = _time(bwd, max(1, iters // 2))
            fl = useful_fwd_flops(lengths, B, S, H, D)
            assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
            rows.append({"shape": f"{B}x{S}x{H}x{D}", "layout": layout,
                         "docs_per_row": None if lengths is None else [len(r) for r in lengths],
                         "useful_fraction": fl / useful_fwd_flops(None, B, S, H, D),
                         "fwd_us": round(fwd_us, 2), "bwd_us": round(bwd_us, 2),
                         "fwd_useful_tflops": round(fl / fwd_us / 1e6, 1),
                         "bwd_useful_tflops": round(2.5 * fl / bwd_us / 1e6, 1)})
    return rows


def worker_step(steps: int, warmup: int):
    import torch

    sys.path.insert(0, ROOT)
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.optim import FusedAdam

    torch.manual_seed(0)
    B, S = 8, 1024
    model = BloomForCausalLM(BloomConfig.bloom_560m()).to(torch.bfloat16).cuda()
    opt = FusedAdam(model.parameters(), lr=1e-5)
    ids = torch.randint(0, model.config.vocab_size, (B, S), device="cuda")
    P = torch.arange(S, device="cuda").remainder(256).expand(B, S).contiguous()
    res = {}
    for name, kw in (("unpacked", {}), ("docs256", {"position_ids": P})):
        def step():
            loss = model(ids, labels=ids, **kw).loss
            opt.zero_grad()
            loss.backward()
            opt.step()
            return loss
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        times = []
        for _ in range(steps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            loss = step()
            e.record()
            torch.cuda.synchronize()
            times.append(s.elapsed_time(e))
        assert math.isfinite(loss.item())
        res[name] = {"step_ms_median": round(statistics.median(times), 2), "step_ms": [round(t, 2) for t in times]}
    return res


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    first = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [p.strip() for p in first.split(",")] if first else []
    return {"gpu": parts[0] if parts else None, "power_limit": parts[1] if len(parts) > 1 else None,
            "max_sm_clock": parts[2] if len(parts) > 2 else None}


def _child(args, ext: str):
    env = dict(os.environ)
    env["PIPEGOOSE_B200_EXT"] = ext
    cmd = [sys.executable, os.path.abspath(__file__)] + args
    res = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"worker failed: {' '.join(args)} (PIPEGOOSE_B200_EXT={ext!r})")
    return json.loads(res.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", help="JSON file to write the results to (required)")
    ap.add_argument("--ab", default="", help="name of a second extension build to time the unpacked rows with")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--worker", choices=["kernels", "step"], help=argparse.SUPPRESS)
    ap.add_argument("--layouts", default=",".join(LAYOUTS), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker == "kernels":
        print(json.dumps(worker_kernels(a.layouts.split(","), a.iters)))
        return
    if a.worker == "step":
        print(json.dumps(worker_step(a.steps, a.warmup)))
        return

    if not a.out:
        ap.error("--out is required")
    card = _card()
    rows = []
    for r in range(a.rounds):
        builds = [("this", "")] + ([(a.ab, a.ab)] if a.ab else [])
        if r % 2:
            builds.reverse()
        for label, ext in builds:
            layouts = LAYOUTS if ext == "" else ["unpacked"]
            for row in _child(["--worker", "kernels", "--iters", str(a.iters), "--layouts", ",".join(layouts)], ext):
                rows.append(dict(row, build=label, round=r))
            print(f"round {r} build {label}: {len(layouts)} layouts", flush=True)
    summary = {}
    for row in rows:
        key = f"{row['shape']} {row['layout']} {row['build']}"
        summary.setdefault(key, {"fwd_us": [], "bwd_us": [], "useful_fraction": row["useful_fraction"]})
        summary[key]["fwd_us"].append(row["fwd_us"])
        summary[key]["bwd_us"].append(row["bwd_us"])
    for key, v in summary.items():
        shape = [int(x) for x in key.split()[0].split("x")]
        fl = v["useful_fraction"] * useful_fwd_flops(None, *shape)
        v["fwd_us_median"] = statistics.median(v["fwd_us"])
        v["bwd_us_median"] = statistics.median(v["bwd_us"])
        v["fwd_useful_tflops"] = round(fl / v["fwd_us_median"] / 1e6, 1)
        v["bwd_useful_tflops"] = round(2.5 * fl / v["bwd_us_median"] / 1e6, 1)
        print(f"{key:40s} fwd {v['fwd_us_median']:9.1f} us {v['fwd_useful_tflops']:6.1f} TF/s   "
              f"bwd {v['bwd_us_median']:9.1f} us {v['bwd_useful_tflops']:6.1f} TF/s", flush=True)
    step = _child(["--worker", "step", "--steps", str(a.steps), "--warmup", str(a.warmup)], "")
    print("bloom-560m step (B=8, S=1024):", {k: v["step_ms_median"] for k, v in step.items()}, flush=True)
    result = {"card": card, "shapes_BxSxHxD": [list(s) for s in SHAPES], "iters": a.iters, "rounds": a.rounds,
              "ab_build": a.ab or None, "summary": summary, "runs": rows, "bloom560m_step_B8_S1024": step}
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
