"""Speed-of-light table of one training step, from MEASURED inputs only (runs here, no GPU):

    python tools/step_roofline.py <step breakdown .json from tools/step_profile.py> > <table>.md

* kernel times: a per-kernel summary of one profiled step (``tools/step_profile.py --aggregate`` on the GPU);
* denominators: ``MEASURED_PEAKS.json`` at the repository root (copy bandwidth and cuBLAS bf16 throughput measured on the
  same part; ``bf16_tflops``, ``bf16_tflops_sustained``, ``hbm_gbs``);
* numerators: FLOPs / bytes every kernel class MUST do for the benchmark's model and batch (formulas below, nothing
  fitted).

For each class: ideal time = max(FLOPs / sustained bf16, bytes / copy bandwidth), fraction = ideal / measured.  The last
column is what the step would gain if that class alone ran at its roofline.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    if len(sys.argv) < 2:
        raise SystemExit("usage: python tools/step_roofline.py <step breakdown .json>")
    path = sys.argv[1]
    prof = json.load(open(path))
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    tf = peaks["bf16_tflops_sustained"] * 1e12          # FLOP/s, back-to-back cuBLAS bf16 (what a step can sustain)
    tf_burst = peaks["bf16_tflops"] * 1e12
    bw = peaks["hbm_gbs"] * 1e9                         # B/s, device copy (read + write bytes)

    # bloom-560m, the headline config (BASELINE.json): 8 x 1024 tokens per GPU, bf16, Adam, tied embedding
    h, L, H, D, V, B, S = 1024, 24, 16, 64, 250880, 8, 1024
    M = B * S
    n_params = V * h + 2 * h + L * (12 * h * h + 13 * h) + 2 * h            # table + emb LN + blocks + ln_f

    layer_gemm = 2 * M * h * (3 * h + h + 4 * h + 4 * h)                     # qkv, dense, fc1, fc2
    head_gemm = 2 * M * V * h
    gemm_pass = L * layer_gemm + head_gemm                                   # one of: forward / dgrad / wgrad
    attn_fwd = L * (4 * B * H * S * S * D) / 2                               # QK^T + PV, causal half
    attn_bwd = attn_fwd * 2.5                                                # S recompute + dP, dV, dQ, dK

    act = M * h * 2                                                          # one [tokens, h] bf16 activation
    rows = {
        # name: (kernel-name fragments, FLOPs, bytes, note)
        "GEMM forward (NT, 96 layer + lm_head)": (["gemm_bf16_kernel<256, 0, 0"], gemm_pass, 0, "wgmma"),
        "GEMM dgrad (NN)": (["gemm_bf16_kernel<256, 0, 1"], gemm_pass, 0, ""),
        "GEMM wgrad (TN, fp32 main-grad accumulate)": (["gemm_bf16_kernel<256, 1, 1"], gemm_pass, 0, ""),
        "attention forward": (["attention_fwd_kernel"], attn_fwd, L * (3 * act + act), "flash, ALiBi in-kernel"),
        "attention backward (+stats, dQ convert)": (["attention_bwd_kernel", "attention_bwd_prep_kernel", "attention_dq_convert_kernel"],
                                                    attn_bwd, L * (3 * act + 2 * act + 3 * act), ""),
        "Adam (fp32 master + 2 moments, bf16 params, fp32 grads)": (["adam_kernel"], 0, n_params * (4 + 8 + 16 + 2), ""),
        "cross entropy (stats + finalize over bf16 logits)": (["ce_finalize_kernel", "ce_stats_kernel"], 0,
                                                              M * V * 2 * 3, "logits read, read, dlogits written"),
        "LayerNorm forward": (["layernorm_fwd_kernel"], 0, (2 * L + 2) * 2 * act, ""),
        "LayerNorm backward (dx + dgamma/dbeta)": (["layernorm_bwd_dx_kernel", "layernorm_bwd_params_kernel"], 0,
                                                   (2 * L + 2) * (3 * act + 2 * act), "dy, x read twice; dx written"),
        "bias gradients (column sums of dY)": (["colsum_kernel"], 0, L * (3 + 1 + 4 + 1) * act, "re-reads every dY"),
    }

    kernels = prof["kernels"]
    total = prof["total_us"]
    used = set()
    out = []
    out.append(f"# Step roofline: bloom-560m, {B} x {S} tokens, 1 GPU ({os.path.basename(path)})\n")
    out.append(f"Denominators (MEASURED_PEAKS.json): bf16 sustained {peaks['bf16_tflops_sustained']:.0f} TFLOP/s "
               f"(burst {peaks['bf16_tflops']:.0f}), copy bandwidth {peaks['hbm_gbs']:.0f} GB/s.  "
               f"Profiled step: {total / 1e3:.2f} ms in {prof['launches']} launches.\n")
    out.append("| kernel class | launches | measured ms | must-do work | ideal ms | fraction of roofline | step gain at roofline |")
    out.append("|---|---|---|---|---|---|---|")
    ideal_total = 0.0
    measured_total = 0.0
    for name, (frags, flops, nbytes, note) in rows.items():
        us, count = 0.0, 0
        for k in kernels:
            flat = k["name"].replace("(int)", "").replace("(bool)", "")
            if any(f.replace(" ", "") in flat.replace(" ", "") for f in frags):
                us += k["us"]
                count += k["count"]
                used.add(k["name"])
        ideal = max(flops / tf, nbytes / bw) * 1e6
        work = f"{flops / 1e12:.2f} TFLOP" if flops / tf >= nbytes / bw else f"{nbytes / 1e9:.1f} GB"
        if flops and nbytes and flops / tf >= nbytes / bw:
            work += f" (+{nbytes / 1e9:.1f} GB)"
        ideal_total += ideal
        measured_total += us
        out.append(f"| {name} | {count} | {us / 1e3:.2f} | {work} | {ideal / 1e3:.2f} | {ideal / us:.2f} | "
                   f"{(us - ideal) / 1e3:.2f} ms ({(us - ideal) / total * 100:.1f} %) |" if us else f"| {name} | 0 | – | {work} | – | – | – |")
    rest = sum(k["us"] for k in kernels if k["name"] not in used)
    out.append(f"| everything else (embedding backward, small torch ops) | – | {rest / 1e3:.2f} | – | – | – | – |")
    out.append(f"| **sum** | | **{(measured_total + rest) / 1e3:.2f}** | | **{ideal_total / 1e3:.2f}** | "
               f"**{ideal_total / (measured_total + rest):.2f}** | |\n")
    gemm_flops = 3 * gemm_pass
    gemm_us = sum(k["us"] for k in kernels if "gemm_bf16_kernel" in k["name"])
    out.append(f"GEMM classes together: {gemm_flops / 1e12:.1f} TFLOP in {gemm_us / 1e3:.2f} ms = "
               f"{gemm_flops / gemm_us / 1e6:.0f} TFLOP/s ({gemm_flops / gemm_us * 1e6 / tf:.2f} of sustained cuBLAS, "
               f"{gemm_flops / gemm_us * 1e6 / tf_burst:.2f} of burst).  Model FLOPs of the step (GEMM + attention): "
               f"{(gemm_flops + attn_fwd + attn_bwd) / 1e12:.1f} TFLOP -> MFU {(gemm_flops + attn_fwd + attn_bwd) / (total * 1e-6) / tf:.2f} "
               f"of sustained over the profiled step.\n")
    out.append(f"Reading: the step is at {ideal_total / (measured_total + rest):.2f} of the sum of its kernels' rooflines.  The GEMMs "
               f"({gemm_us / total * 100:.0f} % of the step) run at {gemm_flops / gemm_us * 1e6 / tf:.2f} of "
               "back-to-back cuBLAS and hold the largest absolute gain; attention is the furthest from its roofline "
               "(latency-bound: short 1024-token sequences, 64-wide heads) and is the second lever; Adam and the cross entropy "
               "passes are at the copy roofline already (the cross-entropy bytes themselves are the waste: logits written and "
               "re-read); LayerNorm and the bias column sums are small, launch-shaped kernels (13-19 us each) at 0.3-0.5.")
    print("\n".join(out))


if __name__ == "__main__":
    main()
