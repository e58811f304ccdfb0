"""bench.py's contract: our arm runs (here: the CPU dry run on gloo with a tiny model), prints ONE JSON line with the agreed
keys, and spells the benchmark configuration exactly as the reference arm does.  The reference arm's lines for the same
commands (``--impl reference`` with the original pipegoose installed under baseline/_ref) are stored in
tests/golden/bench_reference_cpu.json, so the comparison runs without the original project."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMON = ["--device", "cpu", "--model", "bloom-tiny", "--seq-len", "32", "--batch-per-gpu", "2", "--steps", "2", "--warmup", "3"]
with open(os.path.join(ROOT, "tests", "golden", "bench_reference_cpu.json")) as f:
    REFERENCE = json.load(f)


def _run(extra, env=None, steps=None):
    common = COMMON if steps is None else [a if i == 0 or COMMON[i - 1] != "--steps" else str(steps)
                                           for i, a in enumerate(COMMON)]
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + common + extra, capture_output=True, text=True,
                         timeout=600, cwd=ROOT, env=dict(os.environ, **(env or {})))
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, out.stdout[-2000:] + out.stderr[-2000:]
    return json.loads(lines[0])


def test_layout_and_config_helpers():
    sys.path.insert(0, ROOT)
    import argparse

    import bench

    def args(**kw):
        base = dict(gpus=8, tp=0, pp=1, model="bloom-560m", batch_per_gpu=8, seq_len=1024, microbatches=8, experts=0)
        base.update(kw)
        return argparse.Namespace(**base)

    assert bench.layout_of(args(gpus=1)) == (1, 1, 1)
    assert bench.layout_of(args(gpus=2)) == (2, 1, 1)
    assert bench.layout_of(args(gpus=8)) == (2, 1, 4)                      # BASELINE.json's headline: TP2 x DP4
    assert bench.layout_of(args(gpus=8, tp=8)) == (8, 1, 1)                # config #3 / #4
    assert bench.layout_of(args(gpus=8, tp=2, pp=2)) == (2, 2, 2)          # config #5
    cfg = bench.config_of(args(gpus=8), 2, 1, 4)
    assert cfg["parallelism"] == "tp2dp4+zero1" and cfg["global_batch"] == 64 and cfg["model"] == "bloom-560m"
    assert bench.config_of(args(gpus=8, tp=8, experts=8), 8, 1, 1)["parallelism"] == "tp8dp1+moe8e"


@pytest.mark.parametrize("extra", [["--gpus", "1"], ["--gpus", "2"], ["--gpus", "2", "--hf"]])
def test_both_arms_print_one_json_line_with_the_same_config(extra):
    ours = _run(extra)
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "dtype",
                "data", "config", "e2e", "gpu_launches", "clocks"):
        assert key in ours, key
    assert ours["e2e"]["h2d_bytes_per_step"] > 0 and ours["e2e"]["d2h_bytes_per_step"] == 4
    if "--hf" in extra:
        return
    ref = REFERENCE["gpus" + extra[-1]]
    assert ref["impl"] == "reference"
    assert ref["config"] == ours["config"] and ref["metric"] == ours["metric"]
    if extra[-1] != "1":
        assert ours["numerics_ok"] is True      # the self-check ran (on CPU both engines are the library path)


def test_moe_config_both_arms_and_the_reference_arm_in_bf16():
    """BASELINE.json config #4 shape (Switch-MoE, experts sharded over the tensor group).  The reference arm runs with the
    model cast to bf16 as on the GPU: its router stays fp32 (it casts its own input), everything else must cope."""
    extra = ["--gpus", "2", "--tp", "2", "--experts", "2"]
    ours = _run(extra + ["--no-self-check"])
    ref = REFERENCE["gpus2_tp2_experts2_bf16"]  # --impl reference with PIPEGOOSE_B200_BENCH_CPU_BF16=1
    assert ref["impl"] == "reference" and ref["config"] == ours["config"]
    assert ours["config"]["parallelism"] == "tp2dp1+moe2e"
    for line in (ours, ref):
        assert line["final_loss"] == line["final_loss"] and 0 < line["final_loss"] < 20   # finite, of the order of ln(vocab)


def test_dump_outputs_are_repeatable(tmp_path):
    """--dump-outputs writes what the LAST timed step produced: its loss (the JSON line's final_loss) and a seeded sample
    of the parameters it left behind.  The same arguments give the same arrays; one more timed step changes them."""
    import numpy as np

    def run(tag, steps):
        d = tmp_path / tag
        line = _run(["--gpus", "1", "--dump-outputs", str(d)], steps=steps)
        return line, {name: np.load(d / f"{name}.npy") for name in ("loss", "params_sample")}

    (l0, a), (_, b), (l2, c) = run("a", 2), run("b", 2), run("c", 3)
    for name in ("loss", "params_sample"):
        assert a[name].dtype in (np.float32, np.float64) and a[name].size > 0
        np.testing.assert_array_equal(a[name], b[name])
    assert a["loss"][0] == l0["final_loss"] and c["loss"][0] == l2["final_loss"]
    assert l2["steps"] == 3 and not np.array_equal(a["params_sample"], c["params_sample"])
