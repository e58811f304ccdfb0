"""FP8 (e4m3) paged KV cache on CPU: the quantizer's format, the FP8 decode / prefill references against the fp32
references on dequantized pools (the step's own keys and values exact), and ``ContinuousBatcher(kv_cache_dtype=...)``
on tiny fp32 Bloom and GPT-2 models."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (FP8_MAX, PAGE_SIZE, alibi_paged_decode_attention_reference,
                                          alibi_paged_prefill_attention_reference, dequantize_kv,
                                          fp8_prefill_staging, paged_kv_dequantize_reference, paged_kv_write,
                                          quantize_kv)
from pipegoose_b200.serving import ContinuousBatcher

FP8 = torch.float8_e4m3fn


def test_quantizer_format():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(50, 80, generator=g) * torch.logspace(-6, 6, 50).view(-1, 1)
    x[3] = 0.0                                                   # zero row
    x[4, 7] = 1e4                                                # one large outlier
    x[5] = -0.0
    codes, scales = quantize_kv(x.to(torch.bfloat16))
    assert codes.dtype == FP8 and scales.dtype == torch.float32 and scales.shape == (50,)
    c = codes.float()
    nonzero = [r for r in range(50) if r not in (3, 5)]
    assert torch.equal(c[nonzero].abs().amax(-1), torch.full((48,), FP8_MAX))
    for r in (3, 5):
        assert torch.equal(codes[r].view(torch.uint8), torch.zeros(80, dtype=torch.uint8)) and scales[r] == 0
    xb = x.to(torch.bfloat16).float()
    deq = dequantize_kv(codes, scales)
    bound = xb.abs() * 2.0 ** -4 + scales.view(-1, 1) * 2.0 ** -9
    assert ((xb - deq).abs() <= bound).all()


def _fp8_case(H, D, lengths, seed):
    """Random values quantized into FP8 pools with a shuffled table; NaN codes and scales in every other slot."""
    g = torch.Generator().manual_seed(seed)
    need = [(n - 1) // PAGE_SIZE + 1 for n in lengths]
    num_pages = sum(need) + 3
    perm = torch.randperm(num_pages, generator=g).tolist()
    table = torch.zeros(len(lengths), max(need), dtype=torch.int32)
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan")).to(FP8)
    v_pool = k_pool.clone()
    k_scales = torch.full((num_pages, H, PAGE_SIZE), float("nan"))
    v_scales = k_scales.clone()
    for b, n in enumerate(lengths):
        table[b, :need[b]] = torch.tensor(perm[:need[b]], dtype=torch.int32)
        perm = perm[need[b]:]
        p = torch.arange(n)
        page, off = table[b, p // PAGE_SIZE].long(), p % PAGE_SIZE
        for pool, scales in ((k_pool, k_scales), (v_pool, v_scales)):
            codes, s = quantize_kv(torch.randn(n, H, D, generator=g) * 3)
            pool[page, :, off], scales[page, :, off] = codes, s
    return k_pool, v_pool, k_scales, v_scales, table


def _dequantized(pool, scales):
    return dequantize_kv(pool, scales).nan_to_num(0.0)


@pytest.mark.parametrize("D", [64, 80])
def test_decode_reference_reads_dequantized_keys_and_its_own_key_exactly(D):
    H, lengths = 3, [1, 64, 65, 200]
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, lengths, seed=D)
    qkv = torch.randn(len(lengths), H * 3 * D).to(torch.bfloat16).float()
    pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32)
    slopes = K.alibi_slopes(H)
    k_ref, v_ref = _dequantized(k_pool, k_scales), _dequantized(v_pool, v_scales)
    x = qkv.view(-1, H, 3, D)
    for b, n in enumerate(lengths):                             # what the fp32 reference reads: the exact new key
        page, off = table[b, (n - 1) // PAGE_SIZE].long(), (n - 1) % PAGE_SIZE
        k_ref[page, :, off], v_ref[page, :, off] = x[b, :, 1], x[b, :, 2]
    got = alibi_paged_decode_attention_reference(qkv, k_pool, v_pool, table, pos, max(lengths) - 1, slopes, D,
                                                 k_scales=k_scales, v_scales=v_scales)
    want = alibi_paged_decode_attention_reference(qkv, k_ref, v_ref, table, pos, max(lengths) - 1, slopes, D)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    for b, n in enumerate(lengths):                             # pos's slot holds the quantizer's bits
        page, off = table[b, (n - 1) // PAGE_SIZE].long(), (n - 1) % PAGE_SIZE
        codes, s = quantize_kv(x[b, :, 1])
        assert torch.equal(k_pool[page, :, off].view(torch.uint8), codes.view(torch.uint8))
        assert torch.equal(k_scales[page, :, off], s)


@pytest.mark.parametrize("D", [64, 80])
def test_prefill_reference_reads_new_tokens_exactly(D):
    H = 2
    cached, new = [64, 128, 0], [10, 70, 5]
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, [c + n for c, n in zip(cached, new)], seed=D + 1)
    g = torch.Generator().manual_seed(3)
    qkv = torch.randn(sum(new), H * 3 * D, generator=g).to(torch.bfloat16).float()
    cu = torch.tensor([0, 10, 80, 85], dtype=torch.int32)
    start = torch.tensor(cached, dtype=torch.int32)
    slopes = K.alibi_slopes(H)
    slot = torch.cat([table[r, (torch.arange(c, c + n) // PAGE_SIZE)].long() * PAGE_SIZE
                      + torch.arange(c, c + n) % PAGE_SIZE for r, (c, n) in enumerate(zip(cached, new))])
    k_ref, v_ref = _dequantized(k_pool, k_scales), _dequantized(v_pool, v_scales)
    paged_kv_write(qkv, slot, k_ref, v_ref, D)                  # fp32 pools: the new tokens exact
    got = alibi_paged_prefill_attention_reference(qkv, k_pool, v_pool, table, cu, start, 70, slopes, D,
                                                  k_scales=k_scales, v_scales=v_scales)
    want = alibi_paged_prefill_attention_reference(qkv, k_ref, v_ref, table, cu, start, 70, slopes, D)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def test_staging_plan_and_dequantize_reference():
    H, D = 2, 64
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, [130, 64 + 3], seed=7)
    pages = [table[0, :3].tolist(), table[1, :2].tolist()]
    n, src, dst, slot, st_table = fp8_prefill_staging(pages, [128, 64], [130, 67])
    assert n == 5 and src == pages[0][:2] + pages[1][:1] and dst == [0, 1, 3]
    assert slot == [2 * PAGE_SIZE, 2 * PAGE_SIZE + 1, 4 * PAGE_SIZE, 4 * PAGE_SIZE + 1, 4 * PAGE_SIZE + 2]
    assert st_table == [[0, 1, 2], [3, 4, 0]]
    k_out = torch.full((n, H, PAGE_SIZE, D), float("nan"), dtype=torch.bfloat16)
    v_out = k_out.clone()
    paged_kv_dequantize_reference(k_pool, v_pool, k_scales, v_scales, torch.tensor(src), torch.tensor(dst), k_out,
                                  v_out)
    for s, d in zip(src, dst):
        assert torch.equal(k_out[d], dequantize_kv(k_pool[s], k_scales[s]).to(torch.bfloat16))
        assert torch.equal(v_out[d], dequantize_kv(v_pool[s], v_scales[s]).to(torch.bfloat16))
    with pytest.raises(ValueError, match="whole number of pages"):
        fp8_prefill_staging([[0, 1]], [10], [70])


def test_ops_refuse_fp8_pools_without_scales():
    H, D = 2, 64
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, [10], seed=8)
    qkv = torch.randn(1, H * 3 * D)
    pos = torch.tensor([9], dtype=torch.int32)
    with pytest.raises(ValueError, match="need k_scales"):
        alibi_paged_decode_attention_reference(qkv, k_pool, v_pool, table, pos, 9, K.alibi_slopes(H), D)
    with pytest.raises(ValueError, match="need k_scales"):
        paged_kv_write(qkv, torch.tensor([0]), k_pool, v_pool, D, k_scales=k_scales)
    with pytest.raises(ValueError, match="other pools take none"):
        paged_kv_write(qkv, torch.tensor([0]), k_pool.float(), v_pool.float(), D, k_scales=k_scales,
                       v_scales=v_scales)


# ------------------------------------------------------------------------------------------------------------ engine
def _bloom(n_head=4, hidden=64):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(0)
    return BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=hidden, n_layer=2, n_head=n_head)).eval()


def _gpt2():
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=4, n_positions=512)).eval()


MODELS = {"bloom": _bloom, "gpt2": _gpt2, "bloom_d80": lambda: _bloom(n_head=2, hidden=160)}


def _prompts(seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 512, (150,), generator=g).tolist()
    tail = lambda n: torch.randint(0, 512, (n,), generator=g).tolist()   # noqa: E731
    return [base + tail(10), tail(70), base[:64] + tail(20), base[:130] + tail(3), tail(1)]


@pytest.mark.parametrize("arch", list(MODELS))
@pytest.mark.parametrize("prefix_caching", [False, True])
def test_engine_first_tokens_and_completion(arch, prefix_caching):
    model = MODELS[arch]()
    prompts, news = _prompts(1), [6, 3, 5, 4, 2]
    outs = {}
    for dtype in (None, FP8):
        engine = ContinuousBatcher(model, max_cache_tokens=40 * PAGE_SIZE, max_prefill_tokens=300,
                                   prefix_caching=prefix_caching, kv_cache_dtype=dtype)
        if dtype is not None:
            assert engine.k_pools.dtype == FP8 and engine.k_scales.shape == engine.k_pools.shape[:-1]
        rids = [engine.submit(p, n) for p, n in zip(prompts[:2], news[:2])]
        done = dict(engine.step())                                  # the first two prompts' prefill: no hits
        rids += [engine.submit(p, n) for p, n in zip(prompts[2:], news[2:])]
        done.update(engine.run())
        assert len(engine._free) == engine.num_pages
        outs[dtype] = [done[r] for r in rids]
        if prefix_caching:
            assert engine.cached_prompt_tokens == (1 + 2) * PAGE_SIZE
    for i, (a, b) in enumerate(zip(outs[None], outs[FP8])):
        assert len(b) == len(prompts[i]) + news[i]
        if i < 2 or not prefix_caching:                              # prefills without hits
            assert b[:len(prompts[i]) + 1] == a[:len(prompts[i]) + 1], i


def test_engine_never_writes_shared_pages():
    model = _bloom()
    engine = ContinuousBatcher(model, max_cache_tokens=20 * PAGE_SIZE, prefix_caching=True, kv_cache_dtype=FP8)
    prompts = _prompts(2)
    engine.submit(prompts[0], 2)
    engine.run()
    shared = [p for (key, _), p in engine._index.items()][:2]        # the first two pages of prompts[0]
    before = [t[:, shared].clone() for t in (engine.k_pools, engine.v_pools, engine.k_scales, engine.v_scales)]
    rid = engine.submit(prompts[3], 8)                               # shares two pages with prompts[0]
    engine.run()
    assert engine.cached_prompt_tokens == 2 * PAGE_SIZE
    after = [t[:, shared] for t in (engine.k_pools, engine.v_pools, engine.k_scales, engine.v_scales)]
    for a, b in zip(before, after):
        assert torch.equal(a.view(torch.uint8) if a.dtype == FP8 else a, b.view(torch.uint8) if b.dtype == FP8 else b)
    assert rid is not None


def test_engine_refuses_other_cache_dtypes():
    model = _bloom()
    for dtype in (torch.bfloat16, torch.float8_e5m2, torch.float32, "fp8"):
        with pytest.raises(ValueError, match="kv_cache_dtype"):
            ContinuousBatcher(model, max_cache_tokens=4 * PAGE_SIZE, kv_cache_dtype=dtype)
