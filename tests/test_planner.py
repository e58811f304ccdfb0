"""partitioning/planner.py: the per-rank parameter count is the parallelizers' arithmetic (checked against real sharded
models), the memory terms scale as they should, and the plan ranks runnable layouts with the ones that fit first."""
import pytest
import torch

from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.nn import PipelineParallel, TensorParallel
from pipegoose_b200.partitioning.planner import estimate_memory, live_microbatches, local_param_count, main, plan
from pipegoose_b200.testing.utils import init_parallel_context, spawn

CFG = dict(vocab_size=90, hidden_size=32, n_layer=5, n_head=4)       # 90: padded to 96 at tp 2; 5 blocks over 2 / 3 stages


def run_count(rank, world_size, port, tp, pp):
    ctx = init_parallel_context(rank, world_size, port, tp, pp, 1)
    cfg = BloomConfig(**CFG)
    model = TensorParallel(BloomForCausalLM(cfg), ctx).parallelize()
    if pp > 1:
        model = PipelineParallel(model, num_microbatches=2, parallel_context=ctx).parallelize()
        params = list(model._pg_pipeline_stage.parameters())
    else:
        params = list(model.parameters())
    have = sum(p.numel() for p in {id(p): p for p in params}.values())
    stage = ctx.get_local_rank(ParallelMode.PIPELINE)
    assert have == local_param_count(cfg, tp, pp, stage), (tp, pp, stage, have, local_param_count(cfg, tp, pp, stage))
    est = estimate_memory(cfg, tp, pp, 1, batch_per_replica=4, seq_len=8, n_microbatches=2, stage=stage)
    assert est.n_params_local == have and est.params == 2 * have and est.grads == 4 * have and est.optimizer == 12 * have
    ctx.destroy()


@pytest.mark.parametrize("tp,pp", [(1, 1), (2, 1), (2, 2), (1, 3), (4, 1)])
def test_local_parameter_count_matches_sharded_models(tp, pp):
    spawn(run_count, world_size=tp * pp, tp=tp, pp=pp)


def test_memory_terms_scale():
    cfg = BloomConfig.bloom_560m()
    one = estimate_memory(cfg, 1, 1, 1, 8, 1024)
    assert one.n_params_local == sum(p.numel() for p in _meta_model(cfg).parameters())        # 559 M
    assert 6.0 < one.activations / 2**30 < 7.0 and 7.5 < one.logits / 2**30 < 8.5              # 32 M h bytes per block; 2 x 4.1 GB
    dp4 = estimate_memory(cfg, 1, 1, 4, 8, 1024)
    assert dp4.optimizer * 4 == one.optimizer and dp4.params == one.params and dp4.activations == one.activations
    tp2 = estimate_memory(cfg, 2, 1, 1, 8, 1024)
    assert tp2.params < 0.55 * one.params and tp2.activations < 0.7 * one.activations and tp2.logits < 0.55 * one.logits
    re = estimate_memory(cfg, 1, 1, 1, 8, 1024, recompute="block")
    assert re.activations < 0.12 * one.activations
    # pipeline: 1F1B holds pp - stage micro-batches, GPipe all of them
    assert [live_microbatches("1f1b", 4, s, 8) for s in range(4)] == [4, 3, 2, 1]
    assert live_microbatches("gpipe", 4, 3, 8) == 8 and live_microbatches("1f1b", 1, 0, 8) == 1
    first = estimate_memory(cfg, 1, 4, 1, 8, 1024, n_microbatches=8, stage=0)
    last = estimate_memory(cfg, 1, 4, 1, 8, 1024, n_microbatches=8, stage=3)
    assert first.logits == 0 and last.logits > 0 and first.activations > 3.5 * last.activations


def _meta_model(cfg):
    with torch.device("meta"):
        return BloomForCausalLM(cfg)


def test_plan_orders_layouts_and_respects_the_memory_limit(capsys):
    cfg = BloomConfig.bloom_7b1()
    layouts = plan(cfg, 8, global_batch=8, seq_len=2048)
    assert all(l.tp * l.pp * l.dp == 8 for l in layouts) and all(l.fits for l in layouts)
    assert (layouts[0].tp, layouts[0].pp, layouts[0].dp) == (1, 1, 8)          # everything fits in 80 GB: least communication first
    assert [l.relative_step_time for l in layouts] == sorted(l.relative_step_time for l in layouts)
    # with 24 GiB per GPU only the deeply sharded layouts remain runnable, and they come first
    small = plan(cfg, 8, global_batch=8, seq_len=2048, hbm_bytes=24 * 2**30)
    assert small[0].fits and not small[-1].fits and {(l.tp, l.pp) for l in small if l.fits} <= {(4, 2), (8, 1), (2, 4), (4, 1)}
    assert not any((l.tp, l.pp, l.dp) == (1, 1, 8) and l.fits for l in small)
    # constraints: heads divide by tp, a stage has at least one block, the batch divides over the replicas
    tiny = BloomConfig(vocab_size=64, hidden_size=32, n_layer=2, n_head=2)
    assert all(l.tp <= 2 and l.pp <= 2 for l in plan(tiny, 8, global_batch=8, seq_len=16))
    assert all(l.dp in (1, 2) for l in plan(cfg, 8, global_batch=2, seq_len=2048))
    main(["--model", "bloom_3b", "--gpus", "8", "--global-batch", "16", "--seq-len", "1024"])
    assert "GiB/GPU" in capsys.readouterr().out


def test_parameter_count_of_the_gpt2_family():
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    for cfg in (GPT2Config.gpt2_tiny(), GPT2Config.gpt2()):
        with torch.device("meta"):
            model = GPT2LMHeadModel(cfg)
        have = sum(p.numel() for p in {id(p): p for p in model.parameters()}.values())
        assert local_param_count(cfg, 1, 1, 0) == have, (cfg, have)
    assert abs(local_param_count(GPT2Config.gpt2(), 1, 1, 0) - 124.4e6) < 0.5e6      # "gpt2": 124 M
