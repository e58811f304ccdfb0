"""Chunked prefill in ``ContinuousBatcher`` on the CPU reference paths: the schedule (every running request decodes in
every step, page-aligned chunks, the prompt-token budget), fp32 logits against the model's forward for Bloom and
GPT-2 with and without prefix caching, FP8 pools, and the refusals."""
import pytest
import torch

from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel
from pipegoose_b200.ops.attention import PAGE_SIZE
from pipegoose_b200.serving import ContinuousBatcher

FP8 = torch.float8_e4m3fn


def _model(arch="bloom"):
    torch.manual_seed(0)
    if arch == "bloom":
        return BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=64, n_layer=2, n_head=2)).eval()
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=2, n_positions=1200)).eval()


def _spy(engine):
    """Per step: (running requests before it, decode rows, [(chunk start, chunk end, prompt length)])."""
    log, paged = [], engine.model._paged_logits

    def spy(ids, positions, k_pools, v_pools, **kw):
        n_dec = kw.get("n_dec")
        if n_dec is None:
            log.append((len(engine._running), None, []))
        else:
            cu, st = kw["cu_seqlens"].tolist(), kw["start"].tolist()
            chunks = [(s, s + cu[i + 1] - cu[i]) for i, s in enumerate(st)]
            log.append((n_dec, n_dec, chunks))
        return paged(ids, positions, k_pools, v_pools, **kw)
    engine.model._paged_logits = spy
    return log


def test_long_prompt_is_chunked_while_others_decode():
    model = _model()
    engine = ContinuousBatcher(model, max_cache_tokens=64 * PAGE_SIZE, max_prefill_tokens=256, chunked_prefill=True)
    g = torch.Generator().manual_seed(0)
    short = [engine.submit(torch.randint(0, 512, (n,), generator=g).tolist(), 40) for n in (5, 70, 130)]
    engine.step()                                         # the three short prompts, as chunks of one step
    assert len(engine._running) == 3
    log = _spy(engine)
    long_prompt = torch.randint(0, 512, (1000,), generator=g).tolist()
    rid = engine.submit(long_prompt, 4)
    outs = {}
    while engine.has_work():
        running = len(engine._running)
        before = {r.rid: len(r.tokens) for r in engine._running}
        outs.update(engine.step())
        after = {r.rid: len(r.tokens) for r in engine._running}
        after.update({k: len(v) for k, v in outs.items()})
        assert all(after[k] == before[k] + 1 for k in before)     # every running request emitted a token
        assert log[-1][1] in (None, running)
    chunks = [c for _, _, cs in log for c in cs]
    assert sum(e - s for s, e in chunks) == 1000 and chunks[0][0] == 0
    for (s, e), (s2, _) in zip(chunks, chunks[1:]):
        assert e == s2
    for _, _, cs in log:
        assert sum(e - s for s, e in cs) <= 256
        for s, e in cs:
            assert e % PAGE_SIZE == 0 or e == 1000
    assert sum(1 for _, n, cs in log if cs and n == 3) >= 3          # the long prompt shared steps with decodes
    assert len(outs[rid]) == 1004 and all(len(outs[r]) > 0 for r in short)
    assert len(engine._free) == engine.num_pages


def _logits_run(model, prompts, news, **kw):
    """Greedy run; every request's next-token logits in order, and its tokens."""
    engine = ContinuousBatcher(model, max_cache_tokens=40 * PAGE_SIZE, **kw)
    steps, forward = {}, engine._forward

    def spy():
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps.setdefault(r.rid, []).append(logits[j].clone())
        return reqs, logits
    engine._forward = spy
    rids = [engine.submit(p, n) for p, n in zip(prompts[:3], news[:3])]
    engine.step()
    engine.step()
    rids += [engine.submit(p, n) for p, n in zip(prompts[3:], news[3:])]
    outs = engine.run()
    assert len(engine._free) == engine.num_pages
    return [outs[r] for r in rids], [steps[r] for r in rids], engine


@pytest.mark.parametrize("prefix_caching", [False, True])
@pytest.mark.parametrize("arch", ["bloom", "gpt2"])
def test_chunked_logits_match_the_forward(arch, prefix_caching):
    model = _model(arch)
    g = torch.Generator().manual_seed(1)
    system = torch.randint(0, 512, (150,), generator=g).tolist()
    prompts = [system + torch.randint(0, 512, (n,), generator=g).tolist() for n in (3, 200, 40, 90, 1, 300)]
    news = [6, 5, 7, 4, 8, 3]
    outs, steps, engine = _logits_run(model, prompts, news, max_prefill_tokens=128, chunked_prefill=True,
                                      prefix_caching=prefix_caching)
    base, base_steps, base_engine = _logits_run(model, prompts, news, prefix_caching=prefix_caching)
    assert engine.cached_prompt_tokens == base_engine.cached_prompt_tokens
    assert (engine.cached_prompt_tokens > 0) == prefix_caching
    for p, out, got, ref, ref_steps in zip(prompts, outs, steps, base, base_steps):
        with torch.no_grad():
            full = model(torch.tensor([out])).logits[0].float()
        P = len(p)
        for s, lg in enumerate(got):
            assert torch.allclose(lg, full[P - 1 + s], atol=2e-5, rtol=1e-4), (P, s)
        # greedy tokens equal the unchunked engine's until the first near-tie
        for s, lg in enumerate(ref_steps):
            top2 = lg.topk(2).values
            if top2[0] - top2[1] < 1e-3:
                break
            assert out[P + s] == ref[P + s]


def test_fp8_chunks_read_earlier_chunks_dequantized():
    """With FP8 pools a chunked prompt's first-token logits are those of a prefill that runs its chunks one after the
    other through the FP8 reference path (each reading the earlier chunks from the pools, its own tokens exactly),
    and differ from the unchunked prefill's by FP8 rounding only."""
    model = _model()
    g = torch.Generator().manual_seed(2)
    prompt = torch.randint(0, 512, (300,), generator=g).tolist()
    firsts = {}
    for chunked in (False, True):
        engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE, max_prefill_tokens=128,
                                   kv_cache_dtype=FP8, chunked_prefill=chunked)
        forward = engine._forward

        def spy(forward=forward, chunked=chunked):
            reqs, logits = forward()
            if reqs:
                firsts.setdefault(chunked, logits[0].clone())
            return reqs, logits
        engine._forward = spy
        engine.submit(prompt, 2)
        engine.run()
    # the same chunks through the cached-prefix prefill mode, over fresh FP8 pools
    engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE, kv_cache_dtype=FP8)
    pages = list(range(5))
    table = torch.tensor([pages], dtype=torch.int32)
    for s, e in ((0, 128), (128, 256), (256, 300)):
        i32 = lambda x: torch.tensor(x, dtype=torch.int32)   # noqa: E731
        want = model._paged_logits(i32(prompt[s:e]), i32(list(range(s, e))), engine.k_pools, engine.v_pools,
                                   slot=i32([pages[p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE for p in range(s, e)]),
                                   last=i32([e - s - 1]), table=table, cu_seqlens=i32([0, e - s]), start=i32([s]),
                                   max_len=e - s, k_scales=engine.k_scales, v_scales=engine.v_scales)
    assert torch.allclose(firsts[True], want[0].float(), atol=1e-6, rtol=1e-6)
    dist = (firsts[True] - firsts[False]).abs().max() / firsts[False].abs().max()
    assert 0 < dist < 0.05


def test_refusals():
    model = _model()
    with pytest.raises(ValueError, match="at least 64"):
        ContinuousBatcher(model, max_cache_tokens=4096, max_prefill_tokens=63, chunked_prefill=True)
    with pytest.raises(ValueError, match="speculative"):
        ContinuousBatcher(model, max_cache_tokens=4096, chunked_prefill=True, num_speculative_tokens=2)
    ContinuousBatcher(model, max_cache_tokens=4096, max_prefill_tokens=63)          # without chunking: as before
