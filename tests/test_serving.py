"""Continuous batching over a paged KV cache on CPU: the paged decode-attention reference against the contiguous one,
the prefill cache write, and ``ContinuousBatcher`` against ``generate()`` on each prompt alone (tiny fp32 Bloom and
GPT-2 models: the PyTorch references run every step)."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_decode_attention_reference,
                                          alibi_paged_decode_attention, alibi_paged_decode_attention_reference,
                                          paged_kv_write, paged_kv_write_reference)
from pipegoose_b200.serving import ContinuousBatcher


def _scattered(B, H, D, positions, num_pages, seed):
    """Random pools and a shuffled page table: row b owns the pages it needs for positions 0 .. positions[b]."""
    g = torch.Generator().manual_seed(seed)
    k_pool = torch.randn(num_pages, H, PAGE_SIZE, D, generator=g)
    v_pool = torch.randn(num_pages, H, PAGE_SIZE, D, generator=g)
    perm = torch.randperm(num_pages, generator=g).tolist()
    width = max(p // PAGE_SIZE + 1 for p in positions)
    table = torch.full((B, width), 10 ** 6, dtype=torch.int32)      # unused entries: never read
    for b, p in enumerate(positions):
        n = p // PAGE_SIZE + 1
        table[b, :n] = torch.tensor(perm[:n], dtype=torch.int32)
        perm = perm[n:]
    qkv = torch.randn(B, H * 3 * D, generator=g)
    return qkv, k_pool, v_pool, table


def _contiguous(pool, table_row, n):
    """Positions 0 .. n-1 of one table row as a ``[1, H, n, D]`` cache."""
    pages = pool[table_row[: (n - 1) // PAGE_SIZE + 1].long()]                  # [pages, H, 64, D]
    return pages.transpose(0, 1).reshape(pool.shape[1], -1, pool.shape[3])[None, :, :n].clone()


@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_reference_matches_the_contiguous_reference(D):
    B, H = 4, 3
    positions = [0, 63, 64, 200]
    qkv, k_pool, v_pool, table = _scattered(B, H, D, positions, 16, seed=D)
    slopes = K.alibi_slopes(H)
    kc = [_contiguous(k_pool, table[b], p + 1) for b, p in enumerate(positions)]
    vc = [_contiguous(v_pool, table[b], p + 1) for b, p in enumerate(positions)]
    k0, v0 = k_pool.clone(), v_pool.clone()
    pos = torch.tensor(positions, dtype=torch.int32)
    got = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, max(positions) + 5, slopes, D)
    for b, p in enumerate(positions):
        want = alibi_decode_attention_reference(qkv[b:b + 1], kc[b], vc[b], slopes, p, None, D)
        torch.testing.assert_close(got[b:b + 1], want, rtol=1e-5, atol=1e-5)
        page, off = table[b, p // PAGE_SIZE].item(), p % PAGE_SIZE
        x = qkv.view(B, H, 3, D)
        assert torch.equal(k_pool[page, :, off], x[b, :, 1]) and torch.equal(v_pool[page, :, off], x[b, :, 2])
        k0[page, :, off], v0[page, :, off] = x[b, :, 1], x[b, :, 2]
    assert torch.equal(k_pool, k0) and torch.equal(v_pool, v0)      # nothing but the new slots changed


def test_paged_reference_ignores_what_lies_behind_pos():
    B, H, D = 2, 2, 64
    positions = [5, 70]
    qkv, k_pool, v_pool, table = _scattered(B, H, D, positions, 6, seed=1)
    slopes = K.alibi_slopes(H)
    pos = torch.tensor(positions, dtype=torch.int32)
    want = alibi_paged_decode_attention_reference(qkv, k_pool.clone(), v_pool.clone(), table, pos, 127, slopes, D)
    for b, p in enumerate(positions):        # fill every slot a row does not use with NaN
        for q in range(p + 1, (p // PAGE_SIZE + 1) * PAGE_SIZE):
            k_pool[table[b, q // PAGE_SIZE], :, q % PAGE_SIZE] = float("nan")
            v_pool[table[b, q // PAGE_SIZE], :, q % PAGE_SIZE] = float("nan")
    got = alibi_paged_decode_attention_reference(qkv, k_pool, v_pool, table, pos, 127, slopes, D)
    assert torch.equal(got, want)
    with pytest.raises(ValueError, match="max_pos"):
        alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, 128, slopes, D)


def test_paged_kv_write_reference_stores_every_head():
    N, H, D, pages = 7, 3, 80, 4
    g = torch.Generator().manual_seed(2)
    qkv = torch.randn(N, H * 3 * D, generator=g)
    k_pool, v_pool = torch.zeros(pages, H, PAGE_SIZE, D), torch.zeros(pages, H, PAGE_SIZE, D)
    slot = torch.tensor([0, 63, 64, 130, 255, 3, 200], dtype=torch.int32)
    paged_kv_write(qkv, slot, k_pool, v_pool, D)
    x = qkv.view(N, H, 3, D)
    for n, s in enumerate(slot.tolist()):
        assert torch.equal(k_pool[s // PAGE_SIZE, :, s % PAGE_SIZE], x[n, :, 1])
        assert torch.equal(v_pool[s // PAGE_SIZE, :, s % PAGE_SIZE], x[n, :, 2])
    k2, v2 = torch.zeros_like(k_pool), torch.zeros_like(v_pool)
    paged_kv_write_reference(qkv, slot, k2, v2, D)
    assert int((k_pool != 0).sum()) == N * H * D and torch.equal(k2, k_pool) and torch.equal(v2, v_pool)


def _bloom(n_head=4, hidden=64, seed=0):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(seed)
    return BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=hidden, n_layer=2, n_head=n_head)).eval()


def _gpt2(n_positions=256):
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=4,
                                      n_positions=n_positions)).eval()


def _alone(model, prompt, new, **kw):
    return model.generate(torch.tensor(prompt)[None], max_new_tokens=new, **kw)[0].tolist()


@pytest.mark.parametrize("arch", ["bloom", "gpt2", "bloom_d80"])
def test_engine_matches_generate_on_each_prompt_alone(arch):
    model = {"bloom": _bloom, "gpt2": _gpt2, "bloom_d80": lambda: _bloom(n_head=2, hidden=160)}[arch]()
    g = torch.Generator().manual_seed(3)
    lengths = [5, 70, 1, 130, 33, 64, 9, 100]
    news = [10, 3, 1, 40, 70, 1, 25, 12]
    prompts = [torch.randint(0, 512, (n,), generator=g).tolist() for n in lengths]
    # 6 pages: the 3-page request waits for pages, finished requests' pages are reused
    engine = ContinuousBatcher(model, max_cache_tokens=6 * PAGE_SIZE + 10, max_prefill_tokens=100)
    assert engine.num_pages == 6
    rids, outs = {}, {}
    for i in range(4):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(3):
        outs.update(engine.step())
    for i in range(4, len(prompts)):               # submitted while the others run
        rids[i] = engine.submit(prompts[i], news[i])
    outs.update(engine.run())
    assert sorted(outs) == sorted(rids.values())
    assert len(engine._free) == engine.num_pages
    for i, rid in rids.items():
        assert outs[rid] == _alone(model, prompts[i], news[i]), i


def test_engine_stops_at_eos_and_samples_in_groups():
    model = _bloom()
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, 512, (n,), generator=g).tolist() for n in (12, 40, 7)]
    full = _alone(model, prompts[0], 20)
    eos = full[12 + 3]                       # the fourth new token
    stop = full.index(eos, 12) + 1
    engine = ContinuousBatcher(model, max_cache_tokens=8 * PAGE_SIZE)
    a = engine.submit(prompts[0], 20, eos_token_id=eos)
    # top_k = 1 sampling picks the arg-max: it runs in its own group, with its own parameters
    b = engine.submit(prompts[1], 15, do_sample=True, top_k=1, temperature=0.7)
    c = engine.submit(torch.tensor(prompts[2]), 15, do_sample=True, top_k=1, top_p=0.9)
    outs = engine.run()
    assert outs[a] == full[:stop]
    assert outs[a] == _alone(model, prompts[0], 20, eos_token_id=eos)[:stop]
    assert outs[b] == _alone(model, prompts[1], 15)
    assert outs[c] == _alone(model, prompts[2], 15)


def test_engine_prefill_packing_respects_max_prefill_tokens():
    model = _bloom()
    engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE, max_prefill_tokens=50)
    calls = []
    step = model._paged_logits

    def spy(ids, *args, **kw):
        calls.append((ids.shape[0], kw.get("seg_start") is not None))
        return step(ids, *args, **kw)

    model._paged_logits = spy
    for n in (20, 20, 20, 90, 5):
        engine.submit(list(range(1, n + 1)), 2)
    engine.run()
    prefills = [n for n, pre in calls if pre]
    assert prefills == [40, 20, 90, 5]         # packed up to 50 tokens; a longer prompt runs alone, in order


def test_engine_refusals():
    model = _bloom()
    engine = ContinuousBatcher(model, max_cache_tokens=2 * PAGE_SIZE)
    with pytest.raises(ValueError, match="empty prompt"):
        engine.submit([], 4)
    with pytest.raises(ValueError, match="pages"):
        engine.submit(list(range(100)), 29)          # 129 positions: 3 pages of a 2-page pool
    engine.submit(list(range(100)), 28)              # 128: fits exactly
    with pytest.raises(ValueError, match="max_new_tokens"):
        engine.submit([1], 0)
    with pytest.raises(ValueError, match="no page"):
        ContinuousBatcher(model, max_cache_tokens=PAGE_SIZE - 1)
    gpt2 = ContinuousBatcher(_gpt2(n_positions=64), max_cache_tokens=4 * PAGE_SIZE)
    gpt2.submit(list(range(60)), 5)                  # positions 0 .. 63
    with pytest.raises(ValueError, match="n_positions"):
        gpt2.submit(list(range(60)), 6)

    tp = _bloom()
    tp.tp = object()
    with pytest.raises(ValueError, match="tensor-parallel"):
        ContinuousBatcher(tp, max_cache_tokens=PAGE_SIZE)
    piped = _bloom()
    piped._pg_pipeline_engine = object()
    with pytest.raises(ValueError, match="pipelined"):
        ContinuousBatcher(piped, max_cache_tokens=PAGE_SIZE)
    fused = _bloom()

    class FusedMoE(torch.nn.Module):     # stands in for the fused NVLink MoE layer: not an ExpertLayer
        pass

    fused.transformer.h[1].mlp = FusedMoE()
    with pytest.raises(ValueError, match="fused NVLink MoE"):
        ContinuousBatcher(fused, max_cache_tokens=PAGE_SIZE)
