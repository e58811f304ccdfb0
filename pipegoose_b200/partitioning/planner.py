"""Which (tensor, pipeline, data) layout fits an H100's 80 GB, and what does each cost?  An analytic planner (the reference
has ``ProfileByMemory`` for pipeline partitions only, partitioning/profile.py; choosing the layout is left to the user).

``estimate_memory`` counts, per rank, for a Bloom-family config:

* **states** — bf16 parameters, fp32 main gradients (the wgrad kernels accumulate into them), fp32 master weights + two
  Adam moments divided by the data-parallel size (ZeRO-1).  Exact: the same arithmetic as the parallelizers (heads /
  columns / rows divided by the tensor group, the vocabulary zero-padded to a multiple of ``8 x tp``, blocks divided over
  the stages, the tied table on the first and last stage) — ``tests/test_planner.py`` compares it with real sharded models;
* **activations** — what the fused sub-layers keep for backward (the ``save_for_backward`` lists of
  ``ops/functional.py``: per block ``x, LN(x) gathered, qkv, attention output, lse`` and ``x, LN(x) gathered, fc1
  pre-activation, GELU output``), times the micro-batches a stage holds in flight under the schedule
  (``scheduler.peak_live_microbatches``); with ``recompute="block"`` only every block's input plus one block's set;
* **logits** — the last stage's ``[tokens, vocab / tp]`` bf16 logits and their gradient (the cross entropy is fused with the
  lm_head, there is no fp32 copy).

``plan`` enumerates the layouts of ``n_gpus``, drops those that cannot run (heads or blocks not divisible) and ranks the
rest: layouts that fit first, then by an estimated relative step time built from two overhead factors (a tensor group
of 2 and data parallelism + ZeRO-1, measured on bloom-560m on an earlier GPU generation and not re-measured on H100; a
pipeline pays its bubble fraction) — a guide to what to measure first, not a substitute for measuring.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

from pipegoose_b200.constants import H100_HBM_BYTES

BF16, FP32 = 2, 4


@dataclass
class MemoryEstimate:
    params: int
    grads: int
    optimizer: int
    activations: int
    logits: int
    total: int
    n_params_local: int

    def gib(self) -> dict:
        return {k: round(getattr(self, k) / 2**30, 3) for k in ("params", "grads", "optimizer", "activations", "logits", "total")}


def _blocks_of_stage(n_layer: int, pp: int, stage: int) -> int:
    """Blocks on ``stage`` (the structural partitioner's rule: as even as possible, earlier stages take the remainder)."""
    base, extra = divmod(n_layer, pp)
    return base + (1 if stage < extra else 0)


def local_param_count(config, tp: int, pp: int, stage: int) -> int:
    """Parameters one rank of ``stage`` holds (the fused model families: Bloom — tied table, embedding LayerNorm, ALiBi —
    and GPT-2 — tied table, learned positions, no embedding LayerNorm)."""
    h, V = config.hidden_size, config.vocab_size
    mult = 8 * tp
    v_local = ((V + mult - 1) // mult * mult // tp) if tp > 1 else V
    block = (3 * h * h + 3 * h) // tp          # qkv weight + bias, column-parallel
    block += h * h // tp + h                   # dense weight (row-parallel) + replicated bias
    block += (4 * h * h + 4 * h) // tp         # fc1
    block += 4 * h * h // tp + h               # fc2
    block += 4 * h                             # two LayerNorms
    n = _blocks_of_stage(config.n_layer, pp, stage) * block
    if stage == 0:
        n += v_local * h                       # token table
        if getattr(config, "embedding_layernorm", True):
            n += 2 * h                         # Bloom: LayerNorm right after the embedding
        if getattr(config, "position_embedding", "alibi") == "learned":
            n += int(getattr(config, "n_positions", 0)) * h      # GPT-2 family: learned absolute positions (replicated)
    if stage == pp - 1:
        n += 2 * h                             # ln_f
        if pp > 1:
            n += v_local * h                   # the tied table's second copy (lm_head) on the last stage
    return n


def live_microbatches(schedule: str, pp: int, stage: int, n_microbatches: int) -> int:
    if pp == 1:
        return 1
    if schedule.lower() in ("1f1b", "one_f_one_b"):
        return min(pp - stage, n_microbatches)
    return n_microbatches                      # GPipe: every forward before the first backward


def estimate_memory(config, tp: int = 1, pp: int = 1, dp: int = 1, batch_per_replica: int = 8, seq_len: int = 1024,
                    n_microbatches: int = 1, stage: int = 0, schedule: str = "1f1b", zero1: bool = True,
                    recompute: Optional[str] = None) -> MemoryEstimate:
    """Bytes on one rank of pipeline ``stage`` (see the module docstring)."""
    recompute = recompute if recompute is not None else getattr(config, "recompute", "none")
    h, H, V = config.hidden_size, config.n_head, config.vocab_size
    n_local = local_param_count(config, tp, pp, stage)
    params = n_local * BF16
    grads = n_local * FP32
    optimizer = 3 * FP32 * n_local // (dp if zero1 else 1)
    m = max(1, n_microbatches if pp > 1 else 1)
    tokens = batch_per_replica * seq_len // m                  # tokens of one micro-batch
    attn = BF16 * (tokens // tp * h + tokens * h + tokens * 3 * h // tp + tokens * h // tp) + FP32 * tokens * H // tp
    mlp = BF16 * (tokens // tp * h + tokens * h + 2 * tokens * 4 * h // tp)
    stats = 2 * 2 * FP32 * tokens // tp                        # mean, rstd of both LayerNorms
    per_block = attn + mlp + stats
    n_blocks = _blocks_of_stage(config.n_layer, pp, stage)
    if recompute == "block":
        per_mb = n_blocks * BF16 * tokens // tp * h + per_block
    else:
        per_mb = n_blocks * per_block
    activations = per_mb * live_microbatches(schedule, pp, stage, m)
    logits = 0
    if stage == pp - 1:
        mult = 8 * tp
        v_local = ((V + mult - 1) // mult * mult // tp) if tp > 1 else V
        logits = 2 * BF16 * tokens * v_local + BF16 * tokens * h * 2       # logits + dlogits, ln_f output (gathered) + input
    total = params + grads + optimizer + activations + logits
    return MemoryEstimate(params, grads, optimizer, activations, logits, total, n_local)


@dataclass
class Layout:
    tp: int
    pp: int
    dp: int
    n_microbatches: int
    worst_stage_bytes: int
    fits: bool
    bubble: float
    relative_step_time: float
    note: str = ""

    def __str__(self):
        return (f"tp{self.tp} pp{self.pp} dp{self.dp}" + (f" ({self.n_microbatches} micro-batches)" if self.pp > 1 else "") +
                f": {self.worst_stage_bytes / 2**30:.1f} GiB/GPU, {'fits' if self.fits else 'DOES NOT FIT'}, "
                f"bubble {self.bubble:.2f}, est. step x{self.relative_step_time:.2f}{' — ' + self.note if self.note else ''}")


# step time relative to one GPU of a TP2 group and of data parallelism (bloom-560m, 8 x 1024 tokens per GPU, not
# re-measured on H100).  Larger tensor groups are extrapolated per doubling; treat them as an ordering, not a prediction.
_TP2_COST, _DP_COST = 1.12, 1.07


def plan(config, n_gpus: int, global_batch: int, seq_len: int, hbm_bytes: int = H100_HBM_BYTES, headroom: float = 0.9,
         max_tp: int = 8, n_microbatches: Optional[int] = None, schedule: str = "1f1b") -> List[Layout]:
    """Every runnable (tp, pp, dp) of ``n_gpus`` GPUs for ``global_batch`` sequences per step, best first."""
    from pipegoose_b200.nn.pipeline_parallel.scheduler import SchedulerType, get_scheduler

    out: List[Layout] = []
    for tp in [t for t in (1, 2, 4, 8, 16) if t <= max_tp and n_gpus % t == 0]:
        if config.n_head % tp:
            continue
        for pp in [p for p in range(1, n_gpus // tp + 1) if (n_gpus // tp) % p == 0]:
            dp = n_gpus // (tp * pp)
            if pp > config.n_layer or global_batch % dp:
                continue
            per_replica = global_batch // dp
            m = n_microbatches or (min(per_replica, 4 * pp) if pp > 1 else 1)
            if pp > 1 and per_replica % m:
                m = max(d for d in range(1, per_replica + 1) if per_replica % d == 0 and d <= 4 * pp)
            if (per_replica // m) * seq_len % tp:
                continue                                   # token-sharded activations: tokens of a micro-batch divide by tp
            worst = max(estimate_memory(config, tp, pp, dp, per_replica, seq_len, m, stage=s, schedule=schedule).total
                        for s in range(pp))
            bubble = 0.0
            if pp > 1:
                kind = SchedulerType.ONE_F_ONE_B if schedule.lower() in ("1f1b", "one_f_one_b") else SchedulerType.GPIPE
                bubble = get_scheduler(kind)(m, pp).bubble_fraction()
            import math

            rel = (_TP2_COST ** math.log2(tp)) * (_DP_COST if dp > 1 else 1.0) / (1.0 - bubble)
            note = ""
            if pp > 1 and per_replica // m * seq_len < 4096:
                note = "small micro-batches: GEMMs below their efficient size"
                rel *= 1.15
            out.append(Layout(tp, pp, dp, m, worst, worst <= headroom * hbm_bytes, bubble, rel, note))
    out.sort(key=lambda l: (not l.fits, l.relative_step_time, l.worst_stage_bytes))
    return out


def main(argv=None) -> None:
    import argparse

    from pipegoose_b200.models.bloom import BloomConfig

    ap = argparse.ArgumentParser(description="rank the (tp, pp, dp) layouts of a Bloom-family model on H100s")
    ap.add_argument("--model", default="bloom_560m", help="a preset of BloomConfig (bloom_560m, bloom_1b7, bloom_3b, bloom_7b1) "
                    "or GPT2Config (gpt2, gpt2_medium, gpt2_large, gpt2_xl)")
    ap.add_argument("--gpus", type=int, default=8)
    ap.add_argument("--global-batch", type=int, default=64, help="sequences per optimizer step")
    ap.add_argument("--seq-len", type=int, default=1024)
    a = ap.parse_args(argv)
    from pipegoose_b200.models.gpt2 import GPT2Config

    family = GPT2Config if a.model.startswith("gpt2") else BloomConfig
    if not hasattr(family, a.model):
        ap.error(f"unknown preset {a.model!r}")
    cfg = getattr(family, a.model)()
    for layout in plan(cfg, a.gpus, a.global_batch, a.seq_len):
        print(layout)


if __name__ == "__main__":   # python -m pipegoose_b200.partitioning.planner --model bloom_7b1 --gpus 8 --global-batch 8 --seq-len 2048
    main()
