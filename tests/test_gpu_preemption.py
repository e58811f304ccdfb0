"""Preemption on the GPU: ``paged_kv_swap_kernel`` against its reference bit for bit and its refusals, and
``ContinuousBatcher(preemption=True)`` on bf16 Bloom and GPT-2 in a pool small enough that requests are swapped out and
recomputed many times: every step's logits against the training forward (over FP8 pools, against a bf16-pool engine
teacher-forced on the same tokens), swapped pages bit for bit across a swap-out and swap-in, and more running rows per
decode step than the reservation engine when requests stop early."""
import pytest
import torch

from pipegoose_b200.ops.attention import PAGE_SIZE, paged_kv_swap, paged_kv_swap_reference, quantize_kv
from pipegoose_b200.serving import ContinuousBatcher

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn
# Largest logit distance of FP8 pools from bf16 pools, over max |logit| (test_gpu_fp8_kv_cache.py's FP8_VS_BF16).
FP8_VS_BF16 = 0.05


def _bits(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def _pools(L, P, H, D, fp8, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.randn(L, P, H, PAGE_SIZE, D, generator=g, device="cuda")
    v = torch.randn(L, P, H, PAGE_SIZE, D, generator=g, device="cuda")
    if not fp8:
        return k.bfloat16(), v.bfloat16(), None, None
    (k, ks), (v, vs) = quantize_kv(k), quantize_kv(v)
    return k, v, ks, vs


def _host(S, L, H, D, dtype, fp8, fill):
    kv = torch.full((S, L, 2, H, PAGE_SIZE, D), fill, dtype=torch.float32).to(dtype).pin_memory()
    return kv, (torch.full((S, L, 2, H, PAGE_SIZE), float(fill)).pin_memory() if fp8 else None)


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_kv_swap_kernel_round_trip_is_the_reference(D, fp8):
    L, P, H, S = 3, 23, 4, 17
    k, v, ks, vs = _pools(L, P, H, D, fp8, seed=D + fp8)
    out = [(19, 4), (2, 16), (7, 0), (11, 9), (0, 5)]           # scattered pages and slots
    host, hs = _host(S, L, H, D, k.dtype, fp8, 3.0)
    want, wants = host.clone(), (hs.clone() if fp8 else None)
    paged_kv_swap(torch.tensor(out, dtype=torch.int32, device="cuda"), k, v, ks, vs, host, hs, to_host=True)
    paged_kv_swap_reference(out, k.cpu(), v.cpu(), *((ks.cpu(), vs.cpu()) if fp8 else (None, None)), want, wants, True)
    torch.cuda.synchronize()
    assert torch.equal(_bits(host), _bits(want))                # named slots hold the pages, the others are unchanged
    if fp8:
        assert torch.equal(hs, wants)
    back = [(5, 4), (22, 16), (13, 0), (1, 9), (8, 5)]          # into other pages of other pools
    k2, v2, ks2, vs2 = _pools(L, P, H, D, fp8, seed=100 + D)
    ref = [t.cpu() for t in (k2, v2)] + ([ks2.cpu(), vs2.cpu()] if fp8 else [None, None])
    paged_kv_swap(back, k2, v2, ks2, vs2, host, hs, to_host=False)
    paged_kv_swap_reference(back, *ref, want, wants, False)
    for got, exp in zip((k2, v2, ks2, vs2), ref):
        if got is not None:
            assert torch.equal(_bits(got.cpu()), _bits(exp))    # named pages restored bit for bit, the others unchanged
    for (p, _), (q, _) in zip(out, back):
        assert torch.equal(_bits(k2[:, q]), _bits(k[:, p])) and torch.equal(_bits(v2[:, q]), _bits(v[:, p]))
        if fp8:
            assert torch.equal(ks2[:, q], ks[:, p]) and torch.equal(vs2[:, q], vs[:, p])


def test_paged_kv_swap_refusals():
    L, P, H, D, S = 2, 4, 2, 64, 3
    k, v, _, _ = _pools(L, P, H, D, False, seed=0)
    host, _ = _host(S, L, H, D, torch.bfloat16, False, 0.0)
    pairs = [(1, 2)]
    with pytest.raises(RuntimeError, match="pinned"):
        paged_kv_swap(pairs, k, v, None, None, torch.zeros_like(host, device="cpu").contiguous(), None, True)
    with pytest.raises(RuntimeError, match="host_kv must be"):
        paged_kv_swap(pairs, k, v, None, None, host[:, :1].contiguous().pin_memory(), None, True)
    with pytest.raises(RuntimeError, match="host_kv must be"):
        paged_kv_swap(pairs, k, v, None, None, host.float().pin_memory(), None, True)
    with pytest.raises(RuntimeError, match="host_kv must be"):
        paged_kv_swap(pairs, k, v, None, None, _host(S, L, H, 80, torch.bfloat16, False, 0.0)[0], None, True)
    k8, v8, ks, vs = _pools(L, P, H, D, True, seed=1)
    host8, hs = _host(S, L, H, D, FP8, True, 0.0)
    with pytest.raises(RuntimeError, match="host_scales"):
        paged_kv_swap(pairs, k8, v8, ks, vs, host8, None, True)
    with pytest.raises(RuntimeError, match="pinned"):
        paged_kv_swap(pairs, k8, v8, ks, vs, host8, torch.zeros_like(hs, device="cpu").contiguous(), True)
    odd = torch.empty(ks.numel() + 1, device="cuda")[1:].view_as(ks).copy_(ks)    # contiguous, 4 bytes off 16
    with pytest.raises(RuntimeError, match="scales must be 16B aligned"):
        paged_kv_swap(pairs, k8, v8, odd, vs, host8, hs, True)
    with pytest.raises(ValueError, match="outside"):
        paged_kv_swap([(P, 0)], k, v, None, None, host, None, True)


# ------------------------------------------------------------------------------------------------------------ engine
def _bloom(hidden, n_head, n_layer=2, vocab=4096, seed=0):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(seed)
    model = BloomForCausalLM(BloomConfig(vocab_size=vocab, hidden_size=hidden, n_layer=n_layer, n_head=n_head))
    return model.to(torch.bfloat16).cuda().eval()


def _gpt2(hidden, n_head, n_layer=2, vocab=4096, seed=0):
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(seed)
    model = GPT2LMHeadModel(GPT2Config(vocab_size=vocab, hidden_size=hidden, n_layer=n_layer, n_head=n_head,
                                       n_positions=256))
    return model.to(torch.bfloat16).cuda().eval()


def _workload(seed=7, n=12):
    """Prompts of 1 .. 119 tokens (one of 64: its first decode starts a page) and 20 .. 129 new tokens."""
    g = torch.Generator().manual_seed(seed)
    lengths = [int(x) for x in torch.randint(1, 120, (n,), generator=g)]
    lengths[3] = 64
    news = [int(x) for x in torch.randint(20, 130, (n,), generator=g)]
    prompts = [torch.randint(0, 4096, (P,), generator=g).tolist() for P in lengths]
    return prompts, news


def _serve(engine, prompts, news, eos=None):
    rids, outs = {}, {}
    for i in range(len(prompts) // 2):
        rids[i] = engine.submit(prompts[i], news[i], eos_token_id=None if eos is None else eos[i])
    for _ in range(4):
        outs.update(engine.step())
    for i in range(len(prompts) // 2, len(prompts)):
        rids[i] = engine.submit(prompts[i], news[i], eos_token_id=None if eos is None else eos[i])
        outs.update(engine.step())
    outs.update(engine.run())
    return {i: outs[rid] for i, rid in rids.items()}


CONFIGS = {"default": {}, "prefix_caching": dict(prefix_caching=True),
           "chunked_prefill": dict(chunked_prefill=True, max_prefill_tokens=128), "cuda_graphs": dict(cuda_graphs=True)}
ARCHS = [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4), ("gpt2", 256, 4)]


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("arch,hidden,n_head", ARCHS)
def test_engine_with_preemption_matches_training_forward(arch, hidden, n_head, config):
    """Every step's logits of each request against the training forward on its prompt + generated tokens, and its
    tokens against the arg-max wherever the top-2 margin exceeds twice the tolerance.  An 8-page pool and a 3-page host
    pool: requests are both swapped out and recomputed.  FP8 pools: the next test."""
    model = (_bloom if arch == "bloom" else _gpt2)(hidden, n_head)
    prompts, news = _workload()
    engine = ContinuousBatcher(model, max_cache_tokens=8 * PAGE_SIZE, preemption=True,
                               swap_space_tokens=3 * PAGE_SIZE, **CONFIGS[config])
    steps = {}
    forward = engine._forward

    def spy():
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps.setdefault(r.rid, []).append(logits[j].clone())
        return reqs, logits

    engine._forward = spy
    outs = _serve(engine, prompts, news)
    assert len(engine._free) == engine.num_pages and len(engine._host_free) == 3
    assert engine.swapped_out_pages > 0 and engine.swapped_in_pages == engine.swapped_out_pages
    assert engine.recomputed_tokens > 0
    if config == "cuda_graphs":
        assert engine.graph_decode_steps > 0
    for i, out in outs.items():
        P, rid = len(prompts[i]), i
        assert len(out) == P + news[i] and len(steps[rid]) == news[i]
        with torch.no_grad():
            full = model(torch.tensor([out], device="cuda")).logits[0].float()
        scale = full[P - 1:].abs().max().item()
        tol = 3e-2 * scale
        for s, got in enumerate(steps[rid]):
            want = full[P - 1 + s]
            assert (got.float() - want).abs().max().item() <= tol, (i, s, (got.float() - want).abs().max().item(), tol)
            top2 = want.topk(2).values
            if top2[0] - top2[1] > 2 * tol:
                assert out[P + s] == int(want.argmax()), (i, s)
    print(f"\n{arch} hidden={hidden} {config}: {engine.preemptions} preemptions, {engine.swapped_out_pages} pages "
          f"swapped out, {engine.recomputed_tokens} positions recomputed")


@pytest.mark.parametrize("arch,hidden,n_head", ARCHS)
def test_fp8_engine_with_preemption_against_bf16_pools(arch, hidden, n_head):
    """FP8 pools against bf16 pools, as test_gpu_fp8_kv_cache.py compares them: the two engines run in lockstep, the
    FP8 one teacher-forced with the bf16-pool engine's tokens.  Scheduling depends only on tokens and page counts, so
    both serve the same requests in every step, preempting, swapping and recomputing the same ones; every step's logits
    of the FP8 engine lie within FP8_VS_BF16 of max |logit| of the bf16-pool engine's."""
    model = (_bloom if arch == "bloom" else _gpt2)(hidden, n_head)
    prompts, news = _workload()
    engines = {dt: ContinuousBatcher(model, max_cache_tokens=8 * PAGE_SIZE, preemption=True,
                                     swap_space_tokens=3 * PAGE_SIZE, kv_cache_dtype=dt) for dt in (None, FP8)}
    logs = {dt: [] for dt in engines}
    for dt, e in engines.items():
        forward = e._forward

        def spy(forward=forward, log=logs[dt]):
            reqs, logits = forward()
            log.append(([r.rid for r in reqs], None if logits is None else logits.float().clone()))
            return reqs, logits
        e._forward = spy
    picks = {}                                             # (rid, tokens so far) -> the bf16-pool engine's pick
    select = engines[None]._select

    def lead_select(reqs, logits):
        out = select(reqs, logits)
        picks.update({(r.rid, len(r.tokens)): t for r, t in zip(reqs, out)})
        return out
    engines[None]._select = lead_select
    engines[FP8]._select = lambda reqs, logits: [picks[(r.rid, len(r.tokens))] for r in reqs]

    def step():                                            # lockstep: the bf16-pool engine's step first
        for e in engines.values():
            e.step()
    for i in range(len(prompts)):
        for e in engines.values():
            e.submit(prompts[i], news[i])
        if i >= len(prompts) // 2 - 1:
            step()
    while engines[None].has_work():
        step()
    assert not engines[FP8].has_work()
    counters = [{k: getattr(e, k) for k in ("preemptions", "swapped_out_pages", "recomputed_tokens")}
                for e in engines.values()]
    assert counters[0] == counters[1] and counters[0]["swapped_out_pages"] > 0 and counters[0]["recomputed_tokens"] > 0
    assert len(logs[None]) == len(logs[FP8])
    dist = []
    for (r16, l16), (r8, l8) in zip(logs[None], logs[FP8]):
        assert r16 == r8
        if l16 is not None:
            dist.append(((l8 - l16).abs().max() / l16.abs().max()).item())
    print(f"\nfp8 vs bf16 pools under preemption, {arch} hidden={hidden}: max teacher-forced logit distance "
          f"{max(dist):.4f} of max |logit| over {len(dist)} steps; {counters[0]}")
    assert max(dist) < FP8_VS_BF16


@pytest.mark.parametrize("fp8", [False, True])
def test_swapped_pages_come_back_bit_for_bit(fp8):
    """Spy on the engine's swaps: the pages of every swap-in, in their new page ids, equal the pages the same host slots
    received at their swap-out, codes and scales."""
    model = _bloom(256, 4)
    prompts, news = _workload(seed=11)
    engine = ContinuousBatcher(model, max_cache_tokens=8 * PAGE_SIZE, preemption=True,
                               swap_space_tokens=64 * PAGE_SIZE, kv_cache_dtype=FP8 if fp8 else None)
    pools = [t for t in (engine.k_pools, engine.v_pools, engine.k_scales, engine.v_scales) if t is not None]
    saved, checked = {}, [0]
    swap = engine._swap

    def spy(pairs, to_host):
        if to_host:
            for page, slot in pairs:
                saved[slot] = [_bits(t[:, page].clone()) for t in pools]
        swap(pairs, to_host)
        if not to_host:
            for page, slot in pairs:
                for t, before in zip(pools, saved.pop(slot)):
                    assert torch.equal(_bits(t[:, page]), before), (page, slot)
                checked[0] += 1

    engine._swap = spy
    _serve(engine, prompts, news)
    assert checked[0] > 0 and checked[0] == engine.swapped_in_pages and not saved
    assert engine.recomputed_tokens == 0


def test_preemption_holds_more_running_rows_when_requests_stop_early():
    """Sampled requests with a large max_new_tokens over a 64-token vocabulary (a random-init model's distribution is
    near uniform there) stop at their eos_token_id after about 150 tokens on average.  Reserving the whole length at admission
    runs fewer rows per decode step than taking pages as they grow."""
    model = _bloom(256, 4, vocab=64)
    g = torch.Generator().manual_seed(5)
    n, new, eos = 24, 250, 7
    prompts = [torch.randint(0, 64, (int(P),), generator=g).tolist() for P in torch.randint(16, 100, (n,), generator=g)]

    def occupancy(**kw):
        engine = ContinuousBatcher(model, max_cache_tokens=24 * PAGE_SIZE,
                                   generator=torch.Generator(device="cuda").manual_seed(0), **kw)
        rows = []
        forward = engine._forward

        def spy():
            if not engine._admitted:
                rows.append(len(engine._running))
            return forward()

        engine._forward = spy
        rids = [engine.submit(p, new, do_sample=True, eos_token_id=eos) for p in prompts]
        outs = engine.run()
        assert all(outs[r][-1] == eos or len(outs[r]) == len(p) + new for r, p in zip(rids, prompts))
        mean_len = sum(len(outs[r]) - len(p) for r, p in zip(rids, prompts)) / n
        return sum(rows) / len(rows), mean_len, engine

    rows_reserved, len_reserved, _ = occupancy()
    rows_grown, len_grown, engine = occupancy(preemption=True)
    print(f"\nmean running rows per decode step: reservation {rows_reserved:.2f}, preemption {rows_grown:.2f} "
          f"({engine.preemptions} preemptions); mean generated length {len_reserved:.1f} / {len_grown:.1f}")
    assert len_reserved < 0.8 * new and len_grown < 0.8 * new
    assert rows_grown > rows_reserved
