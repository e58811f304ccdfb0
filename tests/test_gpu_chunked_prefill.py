"""Chunked prefill on the GPU: ``ContinuousBatcher(chunked_prefill=True)`` against the training forward
(teacher-forced), with bf16 and FP8 pools."""
import pytest
import torch

from pipegoose_b200.ops.attention import PAGE_SIZE

pytestmark = pytest.mark.gpu

FP8 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------------------ engine
def _model(arch, hidden, n_head):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    if arch == "bloom":
        model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head))
    else:
        model = GPT2LMHeadModel(GPT2Config(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head,
                                           n_positions=512))
    return model.to(torch.bfloat16).cuda().eval()


def _moe_bloom():
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.nn import ExpertParallel
    from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer
    from pipegoose_b200.nn.expert_parallel.routers import Top2Router
    from pipegoose_b200.testing.utils import find_free_port, init_parallel_context

    ctx = init_parallel_context(0, 1, find_free_port(), 1, 1, 1, backend="nccl")
    torch.manual_seed(0)
    model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=256, n_layer=2, n_head=4))
    model = ExpertParallel(model, 4, mapping=[1], router=Top2Router(None, 4, 256), parallel_context=ctx,
                           fused=False).parallelize()
    assert type(model.transformer.h[1].mlp) is ExpertLayer
    return model.to(torch.bfloat16).cuda().eval(), ctx


def _workload(seed=11):
    """Twelve requests that start with one of two shared system prompts (130 / 200 tokens) and the prompt lengths
    they end at (up to 320 tokens: chunks of 128 split most of them)."""
    g = torch.Generator().manual_seed(seed)
    systems = [torch.randint(0, 4096, (n,), generator=g).tolist() for n in (130, 200)]
    prompts, news = [], []
    for i in range(12):
        n = int(torch.randint(1, 120, (1,), generator=g))
        prompts.append(systems[i % 2] + torch.randint(0, 4096, (n,), generator=g).tolist())
        news.append(int(torch.randint(1, 24, (1,), generator=g)))
    return prompts, news


def _run(engine, prompts, news, feed=None):
    """Submit in waves (four, three steps, then one per step) and run to the end; every request's next-token logits in
    order.  ``feed``: {(rid, tokens so far): token} of another engine's choices, taken instead of this one's."""
    steps, mixed = {}, [0]
    forward, select = engine._forward, engine._select

    def spy():
        mixed[0] += bool(engine._admitted and engine._running)
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps.setdefault(r.rid, []).append(logits[j].clone())
        return reqs, logits
    engine._forward = spy
    if feed is not None:
        engine._select = lambda reqs, logits: [feed[(r.rid, len(r.tokens))] for r in reqs]
    rids, outs = {}, {}
    for i in range(4):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(3):
        outs.update(engine.step())
    for i in range(4, len(prompts)):
        rids[i] = engine.submit(prompts[i], news[i])
        outs.update(engine.step())
    outs.update(engine.run())
    assert len(engine._free) == engine.num_pages
    assert mixed[0] > 0                                   # some steps carried decode tokens and chunks together
    return rids, outs, steps


def _check_chunked_engine(model, prefix_caching):
    """Every step's logits of each request against the training forward on its prompt + generated tokens; tokens
    against the arg-max wherever the top-2 margin exceeds twice the tolerance (the pattern of the prefix-cache
    engine test)."""
    from pipegoose_b200.serving import ContinuousBatcher

    prompts, news = _workload()
    engine = ContinuousBatcher(model, max_cache_tokens=24 * PAGE_SIZE, max_prefill_tokens=128,
                               prefix_caching=prefix_caching, chunked_prefill=True)
    rids, outs, steps = _run(engine, prompts, news)
    assert (engine.cached_prompt_tokens > 0) == prefix_caching
    for i, rid in rids.items():
        P, out = len(prompts[i]), outs[rid]
        assert len(out) == P + news[i] and len(steps[rid]) == news[i]
        with torch.no_grad():
            full = model(torch.tensor([out], device="cuda")).logits[0].float()
        tol = 3e-2 * full[P - 1:].abs().max().item()
        for s, got in enumerate(steps[rid]):
            want = full[P - 1 + s]
            assert (got - want).abs().max().item() <= tol, (i, s, (got - want).abs().max().item(), tol)
            top2 = want.topk(2).values
            if bool(top2[0] - top2[1] > 2 * tol):
                assert out[P + s] == int(want.argmax()), (i, s)


@pytest.mark.parametrize("prefix_caching", [False, True])
@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_chunked_engine_matches_training_forward(arch, hidden, n_head, prefix_caching):
    _check_chunked_engine(_model(arch, hidden, n_head), prefix_caching)


def test_chunked_engine_with_expert_mlps():
    model, ctx = _moe_bloom()
    try:
        _check_chunked_engine(model, prefix_caching=True)
    finally:
        ctx.destroy()


# Largest teacher-forced logit distance between FP8 and bf16 pools over max |logit| of the step: the bound of the FP8
# KV-cache engine test.  With chunking, later chunks of a prompt read earlier ones dequantized as well.
FP8_VS_BF16 = 0.05


@pytest.mark.parametrize("prefix_caching", [False, True])
@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_chunked_fp8_engine_against_bf16_pools(arch, hidden, n_head, prefix_caching):
    """The chunked FP8 engine is fed the chunked bf16-pool engine's tokens; its logits stay within FP8_VS_BF16."""
    from pipegoose_b200.serving import ContinuousBatcher

    model = _model(arch, hidden, n_head)
    prompts, news = _workload(seed=13)
    engines = [ContinuousBatcher(model, max_cache_tokens=24 * PAGE_SIZE, max_prefill_tokens=128,
                                 prefix_caching=prefix_caching, chunked_prefill=True, kv_cache_dtype=dt)
               for dt in (None, FP8)]
    rids16, outs16, steps16 = _run(engines[0], prompts, news)
    feed = {(rid, len(prompts[i]) + s): outs16[rid][len(prompts[i]) + s]
            for i, rid in rids16.items() for s in range(news[i])}
    rids8, outs8, steps8 = _run(engines[1], prompts, news, feed=feed)
    assert outs8 == outs16 and engines[0].cached_prompt_tokens == engines[1].cached_prompt_tokens
    dist = [((l8 - l16).abs().max() / l16.abs().max()).item()
            for rid in rids16.values() for l16, l8 in zip(steps16[rid], steps8[rid])]
    print(f"\nchunked fp8 vs bf16 pools, {arch} D={hidden // n_head} prefix_caching={prefix_caching}: max "
          f"teacher-forced logit distance {max(dist):.4f} of max |logit| over {len(dist)} steps")
    assert max(dist) < FP8_VS_BF16
