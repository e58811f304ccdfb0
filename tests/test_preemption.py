"""Preemption in ``ContinuousBatcher`` on CPU (``preemption=True``: pages taken as sequences grow, requests swapped to a
host pool or recomputed when the pool runs out), through the PyTorch reference of ``paged_kv_swap``: every request's
tokens against ``generate()`` on its prompt alone, with swap only, recompute only and both, with and without prefix
caching, chunked prefill and speculative decoding; beam requests beside preempted ones; and the refusals."""
import functools

import pytest
import torch

from pipegoose_b200.ops.attention import PAGE_SIZE, paged_kv_swap, paged_kv_swap_reference, quantize_kv
from pipegoose_b200.serving import ContinuousBatcher

POOL_PAGES = 6
BIG_HOST = 1 << 14


def _bloom():
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(0)
    return BloomForCausalLM(BloomConfig(vocab_size=512, hidden_size=64, n_layer=2, n_head=4)).eval()


def _gpt2():
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config(vocab_size=512, hidden_size=64, n_layer=2, n_head=4, n_positions=256)).eval()


@functools.lru_cache(maxsize=None)
def _model(arch):
    return _bloom() if arch == "bloom" else _gpt2()


def _workload(repetitive=False, n=8, seed=1):
    """Prompts of 1 .. 139 tokens (one of 64 and one of 128: their first decode starts a page) and 20 .. 89 new tokens:
    at most 4 pages per request, several requests' worth of growth in a pool of ``POOL_PAGES``."""
    g = torch.Generator().manual_seed(seed)
    lengths = [int(x) for x in torch.randint(1, 140, (n,), generator=g)]
    lengths[1], lengths[5] = 64, 128
    news = [int(x) for x in torch.randint(20, 90, (n,), generator=g)]
    if repetitive:
        prompts = [(torch.randint(0, 512, (5,), generator=g).tolist() * 40)[:P] for P in lengths]
    else:
        prompts = [torch.randint(0, 512, (P,), generator=g).tolist() for P in lengths]
    return prompts, news


@functools.lru_cache(maxsize=None)
def _alone(arch, prompt, new):
    return _model(arch).generate(torch.tensor(prompt)[None], max_new_tokens=new)[0].tolist()


def _serve(engine, prompts, news, first=4):
    """Staggered submissions: ``first`` requests, three steps, then the rest; returns ``{index: tokens}``."""
    rids, outs = {}, {}
    for i in range(first):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(3):
        outs.update(engine.step())
    for i in range(first, len(prompts)):
        rids[i] = engine.submit(prompts[i], news[i])
    outs.update(engine.run())
    return {i: outs[rid] for i, rid in rids.items()}


def _check_drained(engine):
    assert len(engine._free) == engine.num_pages
    assert len(engine._host_free) == (0 if engine.host_kv is None else engine.host_kv.shape[0])
    assert not engine._preempted and not engine.has_work()


@pytest.mark.parametrize("prefix_caching", [False, True])
@pytest.mark.parametrize("swap_space_tokens", [0, 2 * PAGE_SIZE, BIG_HOST])
@pytest.mark.parametrize("arch", ["bloom", "gpt2"])
def test_engine_with_preemption_matches_generate(arch, swap_space_tokens, prefix_caching):
    prompts, news = _workload()
    engine = ContinuousBatcher(_model(arch), max_cache_tokens=POOL_PAGES * PAGE_SIZE, preemption=True,
                               swap_space_tokens=swap_space_tokens, prefix_caching=prefix_caching)
    outs = _serve(engine, prompts, news)
    for i, out in outs.items():
        assert out == _alone(arch, tuple(prompts[i]), news[i]), i
    assert engine.preemptions > 0
    if swap_space_tokens:
        assert engine.swapped_out_pages > 0 and engine.swapped_in_pages == engine.swapped_out_pages
    if swap_space_tokens != BIG_HOST:
        assert engine.recomputed_tokens > 0
    else:
        assert engine.recomputed_tokens == 0
    if swap_space_tokens == 0:
        assert engine.swapped_out_pages == 0
    _check_drained(engine)


@pytest.mark.parametrize("swap_space_tokens", [0, BIG_HOST])
@pytest.mark.parametrize("mode", ["chunked", "speculative"])
def test_preemption_with_chunked_prefill_and_speculative_decoding(mode, swap_space_tokens):
    kw = dict(chunked_prefill=True, max_prefill_tokens=PAGE_SIZE) if mode == "chunked" else dict(num_speculative_tokens=4)
    prompts, news = _workload(repetitive=mode == "speculative")
    engine = ContinuousBatcher(_model("bloom"), max_cache_tokens=POOL_PAGES * PAGE_SIZE, preemption=True,
                               swap_space_tokens=swap_space_tokens, **kw)
    outs = _serve(engine, prompts, news)
    for i, out in outs.items():
        assert out == _alone("bloom", tuple(prompts[i]), news[i]), i
    assert engine.preemptions > 0
    if mode == "speculative":
        assert engine.speculative_accepted_tokens > 0
    _check_drained(engine)


def test_beam_request_beside_preempted_requests():
    """Three plain requests with short prompts and 150 new tokens each, then a beam request (6 pages reserved), in a
    10-page pool: the beam request is admitted at once and the plain requests outgrow the pool around it.  It is the
    latest submitted request, so latest-submitted-first would pick it before any plain request if beam requests were
    not excluded from the victims."""
    model = _model("bloom")
    prompts, _ = _workload(n=6)
    beam_prompt = prompts[0][:30]
    prompts = [None] + [p[:10] for p in prompts[2:5]]
    news = [None] + [150] * 3

    def run(**kw):
        engine = ContinuousBatcher(model, **kw)
        victims, beside = [], []
        preempt = engine._preempt

        def spy(r, pairs):
            victims.append(r.rid)
            beside.append(any(x.rid == beam for x in engine._running))
            preempt(r, pairs)

        engine._preempt = spy
        rids = [engine.submit(p, n) for p, n in zip(prompts[1:], news[1:])]
        beam = engine.submit(beam_prompt, 100, num_beams=2, num_return_sequences=2, eos_token_id=3)
        outs = engine.run()
        return engine, beam, engine.hypotheses[beam], victims, beside, [outs[r] for r in rids]

    engine, beam, hyps, victims, beside, outs = run(max_cache_tokens=10 * PAGE_SIZE, preemption=True,
                                                    swap_space_tokens=PAGE_SIZE)
    _, _, want, _, _, _ = run(max_cache_tokens=64 * PAGE_SIZE)
    assert any(beside) and beam not in victims          # plain requests were preempted while the beam request ran
    assert [h for h, _ in hyps] == [h for h, _ in want]
    for (_, a), (_, b) in zip(hyps, want):
        assert a == pytest.approx(b, rel=1e-5, abs=1e-5)
    for i, out in enumerate(outs, 1):
        assert out == _alone("bloom", tuple(prompts[i]), news[i]), i
    _check_drained(engine)


@pytest.mark.parametrize("chunked", [False, True])
def test_no_preemption_in_the_step_after_an_admission(chunked):
    kw = dict(chunked_prefill=True, max_prefill_tokens=PAGE_SIZE) if chunked else {}
    prompts, news = _workload(n=10, seed=3)
    engine = ContinuousBatcher(_model("gpt2"), max_cache_tokens=POOL_PAGES * PAGE_SIZE, preemption=True,
                               swap_space_tokens=PAGE_SIZE, **kw)
    step, admitted, preempted = [0], set(), []
    take, swap_in, preempt = engine._take, engine._swap_in, engine._preempt

    def spy_take(r):
        ok = take(r)
        if ok:
            admitted.add(step[0])
        return ok

    def spy_swap_in(r, pairs):
        ok = swap_in(r, pairs)
        if ok:
            admitted.add(step[0])
        return ok

    engine._take, engine._swap_in = spy_take, spy_swap_in
    engine._preempt = lambda r, pairs: (preempted.append(step[0]), preempt(r, pairs))
    for p, n in zip(prompts, news):
        engine.submit(p, n)
    while engine.has_work():
        step[0] += 1
        engine.step()
    assert preempted and engine.preemptions == len(preempted)
    assert not [s for s in preempted if s - 1 in admitted]
    _check_drained(engine)


def test_preemption_refusals():
    model = _model("bloom")
    with pytest.raises(ValueError, match="needs preemption=True"):
        ContinuousBatcher(model, max_cache_tokens=4 * PAGE_SIZE, swap_space_tokens=PAGE_SIZE)
    with pytest.raises(ValueError, match="swap_space_tokens must be at least 0"):
        ContinuousBatcher(model, max_cache_tokens=4 * PAGE_SIZE, preemption=True, swap_space_tokens=-1)
    engine = ContinuousBatcher(model, max_cache_tokens=4 * PAGE_SIZE, preemption=True, swap_space_tokens=PAGE_SIZE)
    with pytest.raises(ValueError, match="the pool has 4"):
        engine.submit([1] * 200, 60)
    assert engine.host_kv.shape == (1, 2, 2, 4, PAGE_SIZE, 16)        # whole pages: [slots, n_layer, 2, H, 64, D]


@pytest.mark.parametrize("fp8", [False, True])
def test_paged_kv_swap_reference_round_trip(fp8):
    L, P, H, D, S = 3, 7, 2, 16, 5
    g = torch.Generator().manual_seed(4)
    k, v = torch.randn(L, P, H, PAGE_SIZE, D, generator=g), torch.randn(L, P, H, PAGE_SIZE, D, generator=g)
    ks = vs = hs = None
    if fp8:
        (k, ks), (v, vs) = quantize_kv(k), quantize_kv(v)
        hs = torch.zeros(S, L, 2, H, PAGE_SIZE)
    host = torch.zeros((S, L, 2, H, PAGE_SIZE, D), dtype=k.dtype)
    pairs = [(5, 3), (0, 1), (6, 4)]
    paged_kv_swap(pairs, k, v, ks, vs, host, hs, to_host=True)
    for page, slot in pairs:
        assert torch.equal(host[slot, :, 0].view(torch.uint8 if fp8 else k.dtype),
                           k[:, page].view(torch.uint8 if fp8 else k.dtype))
        assert torch.equal(host[slot, :, 1].view(torch.uint8 if fp8 else k.dtype),
                           v[:, page].view(torch.uint8 if fp8 else k.dtype))
        if fp8:
            assert torch.equal(hs[slot, :, 0], ks[:, page]) and torch.equal(hs[slot, :, 1], vs[:, page])
    assert not host[[0, 2]].view(torch.uint8).any()                  # slots not named stay as they were
    k2, v2 = torch.zeros_like(k), torch.zeros_like(v)
    ks2, vs2 = (torch.zeros_like(ks), torch.zeros_like(vs)) if fp8 else (None, None)
    back = [(1, 3), (2, 1), (4, 4)]
    paged_kv_swap_reference(back, k2, v2, ks2, vs2, host, hs, to_host=False)
    for (page, _), (new, _) in zip(pairs, back):
        for a, b in [(k2, k), (v2, v)] + ([(ks2, ks), (vs2, vs)] if fp8 else []):
            assert torch.equal(a[:, new].view(torch.uint8), b[:, page].view(torch.uint8))
    assert not k2[:, [0, 3, 5, 6]].view(torch.uint8).any()          # pages not named stay as they were
    with pytest.raises(ValueError, match="outside"):
        paged_kv_swap([(7, 0)], k, v, ks, vs, host, hs, to_host=True)
    with pytest.raises(ValueError, match="host_scales"):
        paged_kv_swap(pairs, k, v, ks, vs, host, None if fp8 else torch.zeros(S, L, 2, H, PAGE_SIZE), to_host=True)
