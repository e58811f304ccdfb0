"""Prefix caching on CPU: the paged prefill-attention reference against the contiguous reference, and
``ContinuousBatcher(prefix_caching=True)`` against ``generate()`` on each prompt alone, with its page accounting
(tiny fp32 Bloom and GPT-2 models: the PyTorch references run every step)."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_attention_reference, alibi_paged_prefill_attention,
                                          alibi_paged_prefill_attention_reference)
from pipegoose_b200.serving import ContinuousBatcher


def _prefill_case(H, D, starts, news, seed, spare_pages=3):
    """Full sequences of random qkv, their keys / values stored in shuffled pages of NaN pools (NaN in every slot a
    sequence does not own), and the new rows packed back to back."""
    g = torch.Generator().manual_seed(seed)
    full = [torch.randn(s + n, H * 3 * D, generator=g) for s, n in zip(starts, news)]
    need = [(s + n - 1) // PAGE_SIZE + 1 for s, n in zip(starts, news)]
    num_pages = sum(need) + spare_pages
    perm = torch.randperm(num_pages, generator=g).tolist()
    width = max(need) + 1
    table = torch.full((len(starts), width), 10 ** 6, dtype=torch.int32)     # unused entries: never read
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan"))
    v_pool = k_pool.clone()
    for r, x in enumerate(full):
        table[r, :need[r]] = torch.tensor(perm[:need[r]], dtype=torch.int32)
        perm = perm[need[r]:]
        p = torch.arange(x.shape[0])
        kv = x.view(-1, H, 3, D)
        k_pool[table[r, p // PAGE_SIZE].long(), :, p % PAGE_SIZE] = kv[:, :, 1]
        v_pool[table[r, p // PAGE_SIZE].long(), :, p % PAGE_SIZE] = kv[:, :, 2]
    qkv = torch.cat([x[s:] for x, s in zip(full, starts)])
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32)
    return full, qkv, k_pool, v_pool, table, cu, torch.tensor(starts, dtype=torch.int32)


@pytest.mark.parametrize("D", [64, 80])
def test_paged_prefill_reference_matches_full_sequence(D):
    H = 3
    starts, news = [0, 63, 64, 65, 200], [70, 1, 64, 5, 30]
    full, qkv, k_pool, v_pool, table, cu, start = _prefill_case(H, D, starts, news, seed=D)
    slopes = K.alibi_slopes(H)
    k0, v0 = k_pool.clone(), v_pool.clone()
    got = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, max(news), slopes, D)
    assert torch.isfinite(got).all()
    for r, (s, n) in enumerate(zip(starts, news)):
        want = alibi_attention_reference(full[r], slopes, 1, s + n, H, D)[s:]
        torch.testing.assert_close(got[cu[r]:cu[r + 1]], want, rtol=1e-5, atol=1e-5)
    assert torch.equal(k_pool.isnan(), k0.isnan()) and torch.equal(k_pool.nan_to_num(), k0.nan_to_num())
    assert torch.equal(v_pool.nan_to_num(), v0.nan_to_num())       # the op does not write the pools


def test_paged_prefill_refusals():
    H, D = 2, 64
    _, qkv, k_pool, v_pool, table, cu, start = _prefill_case(H, D, [0, 64], [10, 3], seed=1)
    slopes = K.alibi_slopes(H)
    with pytest.raises(ValueError, match="longest sequence"):
        alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, 9, slopes, D)
    with pytest.raises(ValueError, match="longest sequence"):
        alibi_paged_prefill_attention_reference(qkv, k_pool, v_pool, table, cu, start, 9, slopes, D)
    with pytest.raises(ValueError, match="max_len"):
        alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, table.shape[1] * PAGE_SIZE + 1, slopes, D)
    q96 = torch.zeros(13, H * 3 * 96)
    pool96 = torch.zeros(4, H, PAGE_SIZE, 96)
    for op in (alibi_paged_prefill_attention, alibi_paged_prefill_attention_reference):
        with pytest.raises(ValueError, match="head size"):
            op(q96, pool96, pool96.clone(), table, cu, start, 10, slopes, 96)


# ------------------------------------------------------------------------------------------------------------ engine
def _bloom(n_head=4, hidden=64, seed=0):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(seed)
    return BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=hidden, n_layer=2, n_head=n_head)).eval()


def _gpt2(n_positions=512):
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=4,
                                      n_positions=n_positions)).eval()


MODELS = {"bloom": _bloom, "gpt2": _gpt2, "bloom_d80": lambda: _bloom(n_head=2, hidden=160)}


def _alone(model, prompt, new):
    return model.generate(torch.tensor(prompt)[None], max_new_tokens=new)[0].tolist()


def _hits(prompt, indexed):
    """Hand count of the pages a prompt reuses: its leading full pages found among ``indexed`` token prefixes,
    at most ``(len - 1) // 64``."""
    n = 0
    while n < (len(prompt) - 1) // PAGE_SIZE and tuple(prompt[:(n + 1) * PAGE_SIZE]) in indexed:
        n += 1
    return n


def _watch(engine):
    """After every step: no page is held by two requests unless it is an indexed full page, reference counts equal
    the holders, and no held page is on the free list."""
    step = engine.step

    def checked():
        out = step()
        holders = {}
        for r in list(engine._admitted) + engine._running:
            for p in r.pages:
                holders[p] = holders.get(p, 0) + 1
        for p, n in holders.items():
            assert engine._refs[p] == n and p not in engine._free
            if n > 1:
                assert p in engine._page_key
        assert len(engine._free) + len(holders) == engine.num_pages
        return out

    engine.step = checked
    return engine


@pytest.mark.parametrize("arch", list(MODELS))
def test_cached_engine_matches_generate_on_each_prompt_alone(arch):
    model = MODELS[arch]()
    g = torch.Generator().manual_seed(5)
    base = torch.randint(0, 512, (200,), generator=g).tolist()

    def tail(n):
        return torch.randint(0, 512, (n,), generator=g).tolist()

    # prompts sharing 0, 63, 64, 65, 128 and 200 tokens with `base`; one of exactly 128 tokens (its two pages cached:
    # only the first is reused, its last token recomputed)
    prompts = [base + tail(10), tail(70), base[:63] + tail(40), base[:64] + tail(20), base[:65] + tail(3),
               base[:128] + tail(1), base + tail(5), base[:128]]
    news = [6, 3, 5, 4, 7, 2, 3, 4]
    engine = _watch(ContinuousBatcher(model, max_cache_tokens=40 * PAGE_SIZE, max_prefill_tokens=300,
                                      prefix_caching=True))
    rids = {0: engine.submit(prompts[0], news[0]), 1: engine.submit(prompts[1], news[1])}
    outs = dict(engine.step())          # prefill of the first two; `base`'s three full pages are indexed
    for i in range(2, len(prompts)):
        rids[i] = engine.submit(prompts[i], news[i])
    outs.update(engine.run())
    assert len(engine._free) == engine.num_pages
    for i, rid in rids.items():
        assert outs[rid] == _alone(model, prompts[i], news[i]), i
    indexed = {tuple(base[:k * PAGE_SIZE]) for k in (1, 2, 3)}
    want = sum(_hits(p, indexed) for p in prompts[2:]) * PAGE_SIZE
    assert want == (0 + 1 + 1 + 2 + 3 + 1) * PAGE_SIZE
    assert engine.cached_prompt_tokens == want


def test_same_prompt_in_successive_steps_and_a_follow_up_turn():
    model = _bloom()
    g = torch.Generator().manual_seed(6)
    first = torch.randint(0, 512, (150,), generator=g).tolist()
    engine = _watch(ContinuousBatcher(model, max_cache_tokens=30 * PAGE_SIZE, prefix_caching=True))
    a = engine.submit(first, 60)
    outs = dict(engine.step())
    b = engine.submit(first, 10)                     # the same prompt, one step later: its two full pages are reused
    outs.update(engine.step())
    assert engine.cached_prompt_tokens == 2 * PAGE_SIZE
    outs.update(engine.run())
    assert outs[a] == _alone(model, first, 60) and outs[b] == _alone(model, first, 10)
    # a follow-up turn repeats the conversation (prompt + output) and adds to it: the pages the generated tokens
    # filled were indexed when the request finished (positions up to len - 2 = 208 are cached: 3 full pages)
    follow = outs[a] + torch.randint(0, 512, (30,), generator=g).tolist()
    before = engine.cached_prompt_tokens
    c = engine.submit(follow, 8)
    outs.update(engine.run())
    assert engine.cached_prompt_tokens - before == 3 * PAGE_SIZE
    assert outs[c] == _alone(model, follow, 8)
    assert len(engine._free) == engine.num_pages


def test_eviction_is_least_recently_freed_first():
    model = _bloom()
    g = torch.Generator().manual_seed(7)
    p1, p2 = (torch.randint(0, 512, (129,), generator=g).tolist() for _ in range(2))
    engine = _watch(ContinuousBatcher(model, max_cache_tokens=6 * PAGE_SIZE, prefix_caching=True))
    a = engine.submit(p1, 2)                          # 3 pages: positions 0 .. 129
    engine.run()
    b = engine.submit(p2, 2)                          # 3 more: every page of the pool has been used once
    engine.run()
    assert len(engine._index) == 4 and len(engine._free) == engine.num_pages
    # the pool keeps both prompts' pages: p1 is hit whole
    c = engine.submit(p1, 2)
    engine.run()
    assert engine.cached_prompt_tokens == 2 * PAGE_SIZE
    # a 4-page request takes the least recently freed pages: p2's (freed before p1's second use), and the unindexed
    # tail page of p1's second use; p1's prefix stays
    engine.submit(torch.randint(0, 512, (10,), generator=g).tolist(), 200)
    engine.run()
    before = engine.cached_prompt_tokens
    f = engine.submit(p1, 1)
    outs = engine.run()
    assert engine.cached_prompt_tokens == before + 2 * PAGE_SIZE
    assert outs[f] == _alone(model, p1, 1)
    e = engine.submit(p2, 1)                          # evicted: no hit
    outs = engine.run()
    assert engine.cached_prompt_tokens == before + 2 * PAGE_SIZE
    assert outs[e] == _alone(model, p2, 1)
    assert len(engine._free) == engine.num_pages
    del a, b, c


def test_admission_with_hits_on_a_nearly_full_pool():
    model = _bloom()
    g = torch.Generator().manual_seed(8)
    shared = torch.randint(0, 512, (128,), generator=g).tolist()
    engine = _watch(ContinuousBatcher(model, max_cache_tokens=5 * PAGE_SIZE, prefix_caching=True))
    a = engine.submit(shared + [1, 2, 3], 60)         # 3 pages, runs long
    engine.step()
    # 2 pages hit (held by a), 1 new needed, 2 free: admitted while a runs
    b = engine.submit(shared + [4], 60)
    engine.step()
    assert engine.cached_prompt_tokens == 2 * PAGE_SIZE and not engine._waiting
    # needs 3 pages with no hit: must wait until a or b finishes, and must not take the shared pages
    c = engine.submit(torch.randint(0, 512, (100,), generator=g).tolist(), 80)
    engine.step()
    assert engine._waiting and engine._waiting[0].rid == c
    outs = engine.run()
    assert sorted(outs) == [a, b, c] and len(engine._free) == engine.num_pages
    # the pool is idle and every page free; a request whose hits are all on the free list revives them and still fits
    d = engine.submit(shared + [9], 5 * PAGE_SIZE - 129)
    outs = engine.run()
    assert outs[d] == _alone(model, shared + [9], 5 * PAGE_SIZE - 129)
    assert len(engine._free) == engine.num_pages


def test_default_off_makes_no_hits_and_the_same_calls():
    model = _bloom()
    g = torch.Generator().manual_seed(9)
    base = torch.randint(0, 512, (140,), generator=g).tolist()
    prompts = [base + [1], base + [2], base[:70]]
    calls = []
    step = model._paged_logits

    def spy(ids, *args, **kw):
        calls.append((ids.shape[0], tuple(sorted(k for k, v in kw.items() if v is not None))))
        return step(ids, *args, **kw)

    model._paged_logits = spy
    engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE)
    assert not engine.prefix_caching
    outs = {}
    for p in prompts:
        engine.submit(p, 3)
        outs.update(engine.step())
    outs.update(engine.run())
    assert engine.cached_prompt_tokens == 0
    prefill = ("last", "seg_start", "slot")
    decode = ("max_pos", "table")
    assert calls == [(141, prefill), (141, prefill), (70, prefill), (3, decode), (3, decode)]
    assert len(engine._free) == engine.num_pages
    for i, p in enumerate(prompts):
        assert outs[i] == _alone(model, p, 3)
