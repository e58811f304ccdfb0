"""Beam search in ``ContinuousBatcher`` on CPU: the candidate-choice and page-copy references against brute force, and
the engine against 🤗 ``generate(num_beams=...)`` on the same weights (tiny fp32 Bloom and GPT-2 models: the PyTorch
references run every step), in the default engine, with prefix caching, chunked prefill and FP8 pools."""
import pytest
import torch

from pipegoose_b200.ops.attention import PAGE_SIZE, paged_kv_copy, paged_kv_copy_reference, quantize_kv
from pipegoose_b200.ops.kernels import beam_topk_reference
from pipegoose_b200.serving import ContinuousBatcher

NO_EOS = 10 ** 6          # an eos id outside the vocabulary: 🤗 then never stops early, like eos_token_id=None here


def _brute(logits, scores, cu, k):
    """float64 log_softmax, add, stable descending sort of each request's flat rows * V scores."""
    x = torch.log_softmax(logits.double(), -1) + scores.double().view(-1, 1)
    V, out = x.shape[1], []
    for a, b in zip(cu, cu[1:]):
        flat = x[a:b].reshape(-1)
        idx = torch.sort(flat, descending=True, stable=True).indices[:k]
        out.append([(float(flat[i]), int(i) % V, int(i) // V + a) for i in idx])
    return out


@pytest.mark.parametrize("V", [16, 50, 513])
def test_beam_topk_reference_matches_brute_force(V):
    g = torch.Generator().manual_seed(V)
    rows = [1, 2, 3, 4, 5, 6, 7, 8]
    cu = [0]
    for n in rows:
        cu.append(cu[-1] + n)
    N, k = cu[-1], 16
    logits = torch.randn(N, V, generator=g) * 3
    logits[:, 3] = float("-inf")                           # vocabulary padding
    logits[0] = logits[0, 0]                               # a row of equal logits: ties to the lower token
    logits[0, 3] = float("-inf")
    logits[10, 7] = logits[10, 9] = logits[10].max()       # a tie at the top of a row
    scores = torch.randn(N, generator=g)
    scores[1] = -1e9                                       # 🤗's initial score of all but the first beam
    scores[5:8] = scores[5]                                # equal beams: ties to the lower row
    logits[6] = logits[5]
    got_s, got_t, got_r, lse = beam_topk_reference(logits, scores, cu, k, return_lse=True)
    torch.testing.assert_close(lse, torch.logsumexp(logits.double(), -1).float())
    exact = torch.log_softmax(logits.double(), -1) + scores.double().view(-1, 1)
    for r, want in enumerate(_brute(logits, scores, cu, k)):
        for j, (s, t, n) in enumerate(want):
            tol = 1e-5 * (1 + abs(s))                      # fp32 rounding (at -1e9 it swallows the log-probs)
            got = (int(got_t[r, j]), int(got_r[r, j]))
            if s == float("-inf"):                         # a padding column: the last candidates of a short row
                assert float(got_s[r, j]) == s and float(exact[got[1], got[0]]) == s
                continue
            assert abs(float(got_s[r, j]) - s) <= tol and abs(float(exact[got[1], got[0]]) - s) <= tol, (r, j)
            near = int(((exact[cu[r]:cu[r + 1]] - s).abs() <= 2 * tol).sum())
            if near == 1:                                  # no other candidate within rounding: the same one
                assert got == (t, n), (r, j)
    assert got_t[0].tolist()[:4] == [0, 1, 2, 4]           # the all-equal row 0, without its padding column 3


def test_beam_topk_refuses_k_beyond_the_vocabulary():
    logits = torch.randn(2, 7)
    with pytest.raises(ValueError, match="k must be"):
        beam_topk_reference(logits, torch.zeros(2), [0, 2], 8)
    with pytest.raises(ValueError, match="cu_beams"):
        beam_topk_reference(logits, torch.zeros(2), [0, 1], 2)


@pytest.mark.parametrize("fp8", [False, True])
def test_paged_kv_copy_reference_copies_exactly_the_leading_slots(fp8):
    g = torch.Generator().manual_seed(int(fp8))
    L, pages, H, D = 3, 6, 2, 64
    k = torch.randn(L, pages, H, PAGE_SIZE, D, generator=g)
    v = torch.randn(L, pages, H, PAGE_SIZE, D, generator=g)
    ks = vs = None
    if fp8:
        k, ks = quantize_kv(k)
        v, vs = quantize_kv(v)
    pairs = [(0, 3, 1), (1, 4, 63), (2, 5, 64), (1, 2, 0)]
    k0, v0 = k.clone(), v.clone()
    s0 = (ks.clone(), vs.clone()) if fp8 else None
    paged_kv_copy(pairs, k, v, ks, vs)
    want = [k0.float(), v0.float()] + ([s0[0], s0[1]] if fp8 else [])
    for src, dst, n in pairs:
        for w in want:
            w[:, dst, :, :n] = w[:, src, :, :n]
    got = [k.float(), v.float()] + ([ks, vs] if fp8 else [])
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert torch.equal(k.float()[:, 3, :, 1:], k0.float()[:, 3, :, 1:])     # slots past the count untouched
    k2, v2 = k0.clone(), v0.clone()
    paged_kv_copy_reference(torch.tensor(pairs, dtype=torch.int32), k2, v2, *(s0 if fp8 else (None, None)))
    assert torch.equal(k2.float(), k.float()) and torch.equal(v2.float(), v.float())


def _bloom(ln_gain=1.0):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(0)
    m = BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=64, n_layer=2, n_head=4)).eval()
    with torch.no_grad():
        m.transformer.ln_f.weight.mul_(ln_gain)
    return m


def _gpt2():
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=4, n_positions=400)).eval()


_MODELS = {}


def _model(arch):
    if arch not in _MODELS:
        _MODELS[arch] = {"bloom": _bloom, "gpt2": _gpt2}[arch]()
        _MODELS[arch + "_hf"] = _MODELS[arch].to_hf().eval()
    return _MODELS[arch], _MODELS[arch + "_hf"]


def hf_beams(hf, prompt, new, W, eos, nrs, **kw):
    """🤗 beam search on one prompt: ``[(prompt + tokens, sequences_score)]`` of its nrs best, best first."""
    out = hf.generate(torch.tensor([prompt]), max_new_tokens=new, num_beams=W, num_return_sequences=nrs,
                      eos_token_id=NO_EOS if eos is None else eos, pad_token_id=0, do_sample=False,
                      return_dict_in_generate=True, output_scores=True, **kw)
    res = []
    for j in range(nrs):
        n = int((out.beam_indices[j] >= 0).sum()) if W > 1 else out.sequences.shape[1] - len(prompt)
        res.append((out.sequences[j, :len(prompt) + n].tolist(), float(out.sequences_scores[j]) if W > 1 else None))
    return res


def _greedy_eos(model, prompt):
    """An eos id the beams reach: the fourth token of the greedy continuation."""
    return model.generate(torch.tensor([prompt]), max_new_tokens=6)[0, len(prompt) + 3].item()


def _check(hyps, want, atol=1e-4):
    assert [h[0] for h in hyps] == [w[0] for w in want]
    for (_, s), (_, t) in zip(hyps, want):
        assert abs(s - t) <= atol, (s, t)


_CASES = [   # (arch, prompt length, max_new_tokens, W, length_penalty, early_stopping, num_return_sequences, eos?)
    ("bloom", 1, 70, 2, 1.0, False, 1, False),
    ("bloom", 63, 5, 4, 0.0, True, 4, True),
    ("bloom", 64, 9, 8, 2.0, "never", 8, True),
    ("bloom", 65, 64, 4, -0.5, False, 2, False),
    ("bloom", 130, 12, 2, 1.0, "never", 2, True),
    ("gpt2", 63, 70, 4, 1.0, False, 4, True),
    ("gpt2", 65, 8, 8, -0.5, True, 1, False),
    ("gpt2", 130, 10, 2, 2.0, "never", 2, True),
]
_MODES = ["default", "prefix", "chunked", "fp8"]


def _engine(model, mode, pages=64):
    kw = {"prefix": {"prefix_caching": True}, "chunked": {"chunked_prefill": True, "max_prefill_tokens": 64},
          "fp8": {"kv_cache_dtype": torch.float8_e4m3fn}}.get(mode, {})
    return ContinuousBatcher(model, max_cache_tokens=pages * PAGE_SIZE, **kw)


@pytest.mark.parametrize("mode", _MODES)
@pytest.mark.parametrize("case", _CASES, ids=[f"{c[0]}-P{c[1]}-W{c[3]}-lp{c[4]}-{c[5]}" for c in _CASES])
def test_engine_matches_hf_beam_search(case, mode):
    arch, P, new, W, lp, es, nrs, use_eos = case
    model, hf = _model(arch)
    g = torch.Generator().manual_seed(P * 31 + W)
    prompt = torch.randint(0, 512, (P,), generator=g).tolist()
    eos = _greedy_eos(model, prompt) if use_eos else None
    kw = dict(num_beams=W, length_penalty=lp, early_stopping=es, num_return_sequences=nrs)
    if mode == "fp8":
        ref = _engine(model, "default")
        rr = ref.submit(prompt, new, eos_token_id=eos, **kw)
        ref.run()
        want = ref.hypotheses.pop(rr)
    else:
        want = hf_beams(hf, prompt, new, W, eos, nrs, length_penalty=lp, early_stopping=es)
    engine = _engine(model, mode)
    rids = [engine.submit(prompt, new, eos_token_id=eos, **kw)]
    if mode == "prefix":                                         # a second request takes the first one's pages
        engine.run()
        rids.append(engine.submit(prompt, new, eos_token_id=eos, **kw))
    outs = engine.run()
    for rid in rids:
        hyps = engine.hypotheses.pop(rid)
        assert len(hyps) == nrs
        assert outs.get(rid, hyps[0][0]) == hyps[0][0]
        if mode == "fp8":              # FP8 keys and values: the default engine's scores at a tolerance
            assert abs(hyps[0][1] - want[0][1]) <= 0.05 * (1 + abs(want[0][1]))
        else:
            _check(hyps, want)
    if mode == "prefix" and P > PAGE_SIZE:
        assert engine.cached_prompt_tokens == (P - 1) // PAGE_SIZE * PAGE_SIZE
    assert len(engine._free) == engine.num_pages


def test_num_beams_1_is_greedy():
    model, _ = _model("bloom")
    prompt = list(range(5, 75))
    a, b = _engine(model, "default"), _engine(model, "default")
    ra, rb = a.submit(prompt, 20), b.submit(prompt, 20, num_beams=1)
    assert a.run()[ra] == b.run()[rb]
    assert not b.hypotheses


def test_beam_requests_share_steps_with_greedy_requests():
    model, hf = _model("bloom")
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, 512, (n,), generator=g).tolist() for n in (30, 64, 100, 5, 70)]
    beams = [(0, 2, 40), (1, 4, 12), (2, 8, 6)]               # (prompt, W, max_new_tokens)
    greedy = [(3, 30), (4, 50)]
    for chunked in (False, True):
        kw = {"chunked_prefill": True, "max_prefill_tokens": 128} if chunked else {}
        alone = ContinuousBatcher(model, max_cache_tokens=80 * PAGE_SIZE, **kw)
        ga = [alone.submit(prompts[i], n) for i, n in greedy]
        want = alone.run()
        engine = ContinuousBatcher(model, max_cache_tokens=80 * PAGE_SIZE, **kw)
        rb = [engine.submit(prompts[i], n, num_beams=W, num_return_sequences=W) for i, W, n in beams]
        rg = [engine.submit(prompts[i], n) for i, n in greedy]
        outs = engine.run()
        for a, b in zip(ga, rg):
            assert outs[b] == want[a]
        for rid, (i, W, n) in zip(rb, beams):
            _check(engine.hypotheses.pop(rid), hf_beams(hf, prompts[i], n, W, None, W))
        assert len(engine._free) == engine.num_pages


def test_fork_copies_are_counted_and_reservation_holds():
    """W = 2 over a 65-token prompt, 4 new tokens, no eos: the first step forks the prompt's row, whose page 1 holds
    one position: the second child copies that slot.  Later forks copy iff two beams share a parent (the page holding
    the next write is the parent's alone); those counts come from the beams' parents, recorded here."""
    model, hf = _model("bloom")
    prompt = list(range(100, 165))
    engine = _engine(model, "default", pages=8)
    forks = []
    fork = engine._fork

    def spy(r, running):
        forks.append([p for _, _, p in running])
        return fork(r, running)

    engine._fork = spy
    rid = engine.submit(prompt, 4, num_beams=2, num_return_sequences=2)
    assert engine._waiting[0].pages_needed == 1 + 2 * (2 - 1)
    engine.run()
    _check(engine.hypotheses.pop(rid), hf_beams(hf, prompt, 4, 2, None, 2))
    assert forks[0] == [0, 0]
    assert engine.beam_page_copies == sum(len(f) - len(set(f)) for f in forks)
    assert len(engine._free) == engine.num_pages


def test_refusals():
    model, _ = _model("bloom")
    engine = _engine(model, "default", pages=4)
    for kw, match in [({"num_beams": 0}, "num_beams"), ({"num_beams": 9}, "num_beams"),
                      ({"num_beams": 2, "do_sample": True}, "do_sample"),
                      ({"num_beams": 2, "num_return_sequences": 3}, "num_return_sequences"),
                      ({"num_return_sequences": 2}, "num_return_sequences"),
                      ({"num_beams": 2, "early_stopping": "sometimes"}, "early_stopping"),
                      ({"num_beams": 8, "max_new_tokens": 100}, "num_beams")]:
        kw = dict({"max_new_tokens": 10}, **kw)
        with pytest.raises(ValueError, match=match):
            engine.submit([1, 2, 3], **kw)
    spec = ContinuousBatcher(model, max_cache_tokens=8 * PAGE_SIZE, num_speculative_tokens=2)
    with pytest.raises(ValueError, match="num_beams"):
        spec.submit([1, 2, 3], 5, num_beams=2)
