"""Speculative decoding on CPU: the paged append-attention reference against single-token decode steps, the prompt-
lookup drafter against a brute-force scan, the verification rules (greedy, rejection sampling, truncation), and
``ContinuousBatcher(num_speculative_tokens=k)`` on tiny fp32 Bloom and GPT-2 models."""
import numpy as np
import pytest
import torch
from scipy import stats

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (APPEND_MAX_TOKENS, PAGE_SIZE, alibi_paged_append_attention,
                                          alibi_paged_decode_attention_reference)
from pipegoose_b200.serving import SPEC_NGRAM_SIZES, ContinuousBatcher, _NgramIndex, verify_drafts


def _append_case(H, D, starts, news, seed):
    """Shuffled pages of NaN pools holding each row's first ``starts[r]`` positions, and the rows' new tokens."""
    g = torch.Generator().manual_seed(seed)
    need = [(s + n - 1) // PAGE_SIZE + 1 for s, n in zip(starts, news)]
    num_pages = sum(need) + 2
    perm = torch.randperm(num_pages, generator=g).tolist()
    table = torch.zeros(len(starts), max(need) + 1, dtype=torch.int32)
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan"))
    v_pool = k_pool.clone()
    for r, s in enumerate(starts):
        table[r, :need[r]] = torch.tensor(perm[:need[r]], dtype=torch.int32)
        perm = perm[need[r]:]
        p = torch.arange(s)
        k_pool[table[r, p // PAGE_SIZE].long(), :, p % PAGE_SIZE] = torch.randn(s, H, D, generator=g)
        v_pool[table[r, p // PAGE_SIZE].long(), :, p % PAGE_SIZE] = torch.randn(s, H, D, generator=g)
    qkv = torch.randn(sum(news), H * 3 * D, generator=g)
    cu = torch.tensor([0] + np.cumsum(news).tolist(), dtype=torch.int32)
    return qkv, k_pool, v_pool, table, cu, torch.tensor(starts, dtype=torch.int32)


@pytest.mark.parametrize("D", [64, 80])
def test_append_reference_equals_single_token_decode_steps(D):
    H = 3
    starts, news = [0, 1, 60, 64, 130, 5], [1, 8, 7, 2, 4, 3]        # 60 + 7 and 62..: crossing a page
    qkv, k_pool, v_pool, table, cu, pos = _append_case(H, D, starts, news, seed=D)
    slopes = K.alibi_slopes(H)
    max_pos = max(s + n - 1 for s, n in zip(starts, news))
    k1, v1 = k_pool.clone(), v_pool.clone()
    got = alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, max_pos, slopes, D)
    assert torch.isfinite(got).all()
    for r, (s, n) in enumerate(zip(starts, news)):
        for i in range(n):                                            # one decode step per token, one after another
            row = int(cu[r]) + i
            want = alibi_paged_decode_attention_reference(qkv[row:row + 1], k1, v1, table[r:r + 1],
                                                          torch.tensor([s + i]), s + i, slopes, D)
            torch.testing.assert_close(got[row:row + 1], want, rtol=1e-5, atol=1e-5)
    assert torch.equal(k_pool.isnan(), k1.isnan()) and torch.equal(k_pool.nan_to_num(), k1.nan_to_num())
    assert torch.equal(v_pool.isnan(), v1.isnan()) and torch.equal(v_pool.nan_to_num(), v1.nan_to_num())


def test_append_refusals():
    H, D = 2, 64
    qkv, k_pool, v_pool, table, cu, pos = _append_case(H, D, [3, 70], [2, 9], seed=1)
    slopes = K.alibi_slopes(H)
    with pytest.raises(ValueError, match="1 .. 8 tokens"):
        alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, 80, slopes, D)
    qkv, k_pool, v_pool, table, cu, pos = _append_case(H, D, [3, 70], [2, 5], seed=1)
    with pytest.raises(ValueError, match="last appended position"):
        alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, 73, slopes, D)
    with pytest.raises(ValueError, match="max_pos"):
        alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, table.shape[1] * PAGE_SIZE, slopes, D)
    fp8 = k_pool.to(torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="FP8"):
        alibi_paged_append_attention(qkv, fp8, fp8.clone(), table, cu, pos, 74, slopes, D)
    for bad in (9, -1):
        with pytest.raises(ValueError, match="max_tokens"):
            alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, 74, slopes, D, max_tokens=bad)
    with pytest.raises(ValueError, match="longest row"):
        alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, 74, slopes, D, max_tokens=4)


# ------------------------------------------------------------------------------------------------------------ drafter
def _brute_draft(tokens, k):
    for n in SPEC_NGRAM_SIZES:
        L = len(tokens)
        if L <= n:
            continue
        for i in range(L - n - 1, -1, -1):
            if tokens[i:i + n] == tokens[L - n:]:
                return tokens[i + n:i + n + k]
    return []


@pytest.mark.parametrize("vocab", [3, 6, 50])
def test_incremental_drafter_equals_brute_force(vocab):
    rng = np.random.default_rng(vocab)
    for _ in range(20):
        tokens = rng.integers(0, vocab, int(rng.integers(1, 12))).tolist()
        idx = _NgramIndex()
        for _ in range(60):
            idx.update(tokens)
            k = int(rng.integers(0, 8))
            assert idx.draft(tokens, k) == _brute_draft(tokens, k)
            tokens += rng.integers(0, vocab, int(rng.integers(1, 4))).tolist()


def test_engine_draft_respects_the_budget():
    model = _bloom()
    eng = ContinuousBatcher(model, max_cache_tokens=1024, num_speculative_tokens=7)
    eng.submit([1, 2, 3, 4, 5, 6, 7, 8, 9, 1, 2, 3], max_new_tokens=4)
    r = eng._waiting[0]
    assert eng._draft(r) == [4, 5, 6]                  # budget max_new - generated - 1 = 3
    r.tokens.append(4)
    assert eng._draft(r) == [5, 6]
    r.tokens += [5, 6]
    assert eng._draft(r) == []


# ------------------------------------------------------------------------------------------------------ verification
def _greedy_logits(argmaxes, V=10):
    lg = torch.zeros(len(argmaxes), V)
    lg[torch.arange(len(argmaxes)), torch.tensor(argmaxes)] = 5.0
    return lg


def test_greedy_verification_rules():
    greedy = (False,)
    # request 0: last token 9, drafts [1, 2, 3]; the arg-maxes accept 1 and 2 and replace 3 by 7
    # request 1: last token 4, drafts [5]; accepted, then the bonus arg-max 6
    # request 2: no draft: just the arg-max
    ids = torch.tensor([9, 1, 2, 3, 4, 5, 8])
    lg = _greedy_logits([1, 2, 7, 0, 5, 6, 2])
    out = verify_drafts([greedy] * 3, [[1, 2, 3], [5], []], ids, lg)
    assert out == [[1, 2, 7], [5, 6], [2]]
    lg = _greedy_logits([0, 2, 7, 0, 1, 6, 2])
    assert verify_drafts([greedy] * 3, [[1, 2, 3], [5], []], ids, lg) == [[0], [1], [2]]


def _engine_with(model, prompt, max_new, eos=None, k=3):
    eng = ContinuousBatcher(model, max_cache_tokens=2048, num_speculative_tokens=k)
    rid = eng.submit(prompt, max_new_tokens=max_new, eos_token_id=eos)
    return eng, rid


def test_engine_truncates_at_eos_and_max_new_tokens():
    model = _bloom()
    prompt = [5, 6, 7, 8] * 8
    for max_new in (1, 2, 5, 9):
        eng, rid = _engine_with(model, prompt, max_new)
        out = eng.run()[rid]
        assert len(out) == len(prompt) + max_new
        ref, rref = _engine_with(model, prompt, max_new, k=0)
        assert ref.run()[rref] == out
    eng, rid = _engine_with(model, prompt, 12)
    full = eng.run()[rid]
    eos = full[len(prompt) + 3]
    eng, rid = _engine_with(model, prompt, 12, eos=eos)
    out = eng.run()[rid]
    gen = out[len(prompt):]
    assert gen[-1] == eos and eos not in gen[:-1] and gen == full[len(prompt):len(prompt) + len(gen)]


def _chi2(samples, p):
    """p-value of the samples against the distribution p (bins with p = 0 must stay empty)."""
    counts = np.bincount(samples, minlength=len(p))
    assert counts[p == 0].sum() == 0
    keep = p > 0
    return stats.chisquare(counts[keep], p[keep] / p[keep].sum() * len(samples)).pvalue


@pytest.mark.parametrize("filters", [(1.0, 0, 1.0), (0.7, 4, 1.0), (1.0, 0, 0.8)])
def test_rejection_sampling_keeps_the_distribution(filters):
    from pipegoose_b200.models.bloom import filter_logits

    V, trials = 8, 20000
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(3, V, generator=g) * 1.5
    key = (True,) + filters
    p = filter_logits(logits, *filters).softmax(-1).double().numpy()
    # the drafts: a likely token first, then for row 1 a token that the filters may remove
    d0 = int(np.argsort(p[0])[-2])
    d1 = int(np.argmin(p[1]))
    ids = torch.tensor([0, d0, d1])
    out = verify_drafts([key] * trials, [[d0, d1]] * trials, ids.repeat(trials),
                        logits.repeat(trials, 1), generator=torch.Generator().manual_seed(1))
    first = np.array([o[0] for o in out])
    assert _chi2(first, p[0]) > 1e-3
    second = np.array([o[1] for o in out if o[0] == d0])
    assert _chi2(second, p[1]) > 1e-3
    if p[1][d1] == 0:
        assert all(len(o) < 3 for o in out)                     # a draft of probability 0 is never accepted


# ------------------------------------------------------------------------------------------------------------ engine
def _bloom(n_head=4, hidden=64, seed=0):
    """Weights drawn wider than the default 0.02: the tiny model's greedy outputs then vary instead of repeating one
    token, so verification both accepts and rejects drafts."""
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(seed)
    return BloomForCausalLM(BloomConfig(vocab_size=64, hidden_size=hidden, n_layer=2, n_head=n_head,
                                        initializer_range=0.5)).eval()


def _gpt2():
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=64, hidden_size=64, n_layer=2, n_head=4, n_positions=512,
                                      initializer_range=0.5)).eval()


def _prompts(n, seed=0, vocab=64):
    """Prompts with repeats, so that the drafter finds n-grams."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        base = rng.integers(0, vocab, int(rng.integers(4, 12))).tolist()
        out.append((base * 4)[:int(rng.integers(10, 90))] + rng.integers(0, vocab, 6).tolist())
    return out


def _check_greedy_against_full_forward(model, outs, prompts, rel_tie):
    for toks, prompt in zip(outs, prompts):
        ids = torch.tensor(toks[:-1]).view(1, -1).to(next(model.parameters()).device)
        logits = model(ids).logits[0].float()
        for t in range(len(prompt) - 1, len(toks) - 1):
            top2 = logits[t].topk(2).values
            if toks[t + 1] != int(logits[t].argmax()):
                assert float(top2[0] - top2[1]) < rel_tie * float(top2[0].abs()), (t, toks[t + 1])


@pytest.mark.parametrize("arch", ["bloom", "gpt2"])
def test_greedy_speculative_matches_full_forward_argmax(arch):
    model = _bloom() if arch == "bloom" else _gpt2()
    prompts = _prompts(6)
    eng = ContinuousBatcher(model, max_cache_tokens=64 * 40, num_speculative_tokens=5)
    rids = [eng.submit(p, max_new_tokens=20 + 3 * i) for i, p in enumerate(prompts)]
    outs = eng.run()
    with torch.no_grad():
        _check_greedy_against_full_forward(model, [outs[r] for r in rids], prompts, 1e-4)
    assert eng.speculative_proposed_tokens > eng.speculative_accepted_tokens > 0
    assert len(eng._free) == eng.num_pages


def test_sampled_speculative_engine_runs_and_frees_pages():
    model = _bloom()
    g = torch.Generator().manual_seed(3)
    eng = ContinuousBatcher(model, max_cache_tokens=64 * 40, num_speculative_tokens=4, generator=g)
    prompts = _prompts(5, seed=2)
    rids = [eng.submit(p, max_new_tokens=16, do_sample=True, temperature=0.8, top_k=10 * (i % 2), top_p=0.9)
            for i, p in enumerate(prompts)]
    outs = eng.run()
    assert all(len(outs[r]) == len(p) + 16 for r, p in zip(rids, prompts))
    assert eng.speculative_proposed_tokens > 0
    assert len(eng._free) == eng.num_pages


def test_prefix_cache_reuses_pages_of_a_speculative_request():
    model = _bloom()
    first = ([3, 1, 4, 1, 5, 9, 2, 6] * 12)[:70]
    outs = {}
    for caching in (False, True):
        eng = ContinuousBatcher(model, max_cache_tokens=64 * 20, num_speculative_tokens=6, prefix_caching=caching)
        rid = eng.submit(first, max_new_tokens=90)
        later = eng.run()[rid][:150] + [7, 7]         # reuses the pages the speculative request's tokens filled
        rid = eng.submit(later, max_new_tokens=10)
        outs[caching] = eng.run()[rid]
        if caching:
            assert eng.cached_prompt_tokens >= 128
            assert len(eng._free) == eng.num_pages
    assert outs[True] == outs[False]


def test_speculation_refusals():
    model = _bloom()
    for k in (-1, 8):
        with pytest.raises(ValueError, match="num_speculative_tokens"):
            ContinuousBatcher(model, max_cache_tokens=1024, num_speculative_tokens=k)
    with pytest.raises(ValueError, match="FP8"):
        ContinuousBatcher(model, max_cache_tokens=1024, num_speculative_tokens=2, kv_cache_dtype=torch.float8_e4m3fn)
    assert APPEND_MAX_TOKENS == 8


def test_models_without_an_append_kernel_use_the_reference(monkeypatch):
    """The verify step of a model whose head size has no kernel (here: CPU fp32) runs the reference, never the op that
    dispatches to the kernel."""
    from pipegoose_b200.ops import attention as A

    def kernel_op(*args, **kwargs):
        raise AssertionError("the kernel op was called for a model without a native append path")

    monkeypatch.setattr(A, "alibi_paged_append_attention", kernel_op)
    model = _bloom(n_head=4, hidden=64)
    eng = ContinuousBatcher(model, max_cache_tokens=64 * 10, num_speculative_tokens=3)
    rids = [eng.submit(p, max_new_tokens=12) for p in _prompts(2)]
    outs = eng.run()
    assert all(len(outs[r]) == len(p) + 12 for r, p in zip(rids, _prompts(2)))
    assert eng.speculative_proposed_tokens > 0


def test_accepted_counter_counts_emitted_drafts(monkeypatch):
    from pipegoose_b200 import serving

    model = _bloom()
    prompt = [1, 2, 3, 4, 5, 6, 1, 2]
    eng = ContinuousBatcher(model, max_cache_tokens=1024, num_speculative_tokens=3)
    rid = eng.submit(prompt, max_new_tokens=10, eos_token_id=4)
    eng.step()                                          # prefill: the first new token
    eng._running[0].tokens[-1:] = [3]                   # trailing n-gram [1, 2, 3]: the drafter proposes [4, 5, 6]
    monkeypatch.setattr(serving, "verify_drafts", lambda samplings, drafts, *a: [d + [9] for d in drafts])
    done = eng.step()                                   # every draft accepted; the eos (4) cuts after the first
    assert done and done[0][0] == rid and done[0][1][-1] == 4
    assert (eng.speculative_proposed_tokens, eng.speculative_accepted_tokens) == (3, 1)
