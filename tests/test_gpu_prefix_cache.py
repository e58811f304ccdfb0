"""Prefix caching on the GPU: the paged form of the flash kernel against its fp32 reference (cached prefixes of
different lengths, shuffled pages, NaN outside the valid slots) and against the flash kernel on the same packed
tokens, and ``ContinuousBatcher(prefix_caching=True)`` on bf16 models against the training forward and ``generate()``."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_attention, alibi_paged_prefill_attention,
                                          alibi_paged_prefill_attention_reference, paged_kv_write)

pytestmark = pytest.mark.gpu

STARTS = [0, 64, 1000, 4160]
NEWS = [1, 2, 127, 128, 129, 1000]


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _case(H, D, starts, news, seed, spare_pages=4):
    """NaN pools with random keys / values in every sequence's slots 0 .. start + new - 1 (prefix and new tokens), a
    shuffled page table, and the new tokens' qkv packed back to back."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(s + n - 1) // PAGE_SIZE + 1 for s, n in zip(starts, news)]
    num_pages = sum(need) + spare_pages
    perm = torch.randperm(num_pages, device="cuda", generator=g).to(torch.int32)
    table = torch.full((len(starts), max(need) + 1), -7, dtype=torch.int32, device="cuda")   # never read
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    v_pool = k_pool.clone()
    used = 0
    for r, (s, n) in enumerate(zip(starts, news)):
        table[r, :need[r]] = perm[used:used + need[r]]
        used += need[r]
        p = torch.arange(s + n, device="cuda")
        pages, slots = table[r, p // PAGE_SIZE].long(), p % PAGE_SIZE
        k_pool[pages, :, slots] = torch.randn(s + n, H, D, device="cuda", generator=g).to(torch.bfloat16)
        v_pool[pages, :, slots] = torch.randn(s + n, H, D, device="cuda", generator=g).to(torch.bfloat16)
    qkv = torch.randn(sum(news), H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    return qkv, k_pool, v_pool, table, cu, torch.tensor(starts, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_prefill_kernel_matches_reference(D):
    H = 2
    starts = [STARTS[i % len(STARTS)] for i in range(8)]
    news = [NEWS[(i + D) % len(NEWS)] for i in range(8)]
    qkv, k_pool, v_pool, table, cu, start = _case(H, D, starts, news, seed=D)
    slopes = K.alibi_slopes(H, device="cuda")
    k0, v0 = k_pool.clone(), v_pool.clone()
    out = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, max(news), slopes, D)
    ref = alibi_paged_prefill_attention_reference(qkv.float(), k_pool.float(), v_pool.float(), table, cu, start,
                                                  max(news), slopes, D)
    assert torch.isfinite(out).all()
    for r in range(len(starts)):
        rows = slice(int(cu[r]), int(cu[r + 1]))
        assert _rel(out[rows], ref[rows]) < 1e-2, (starts[r], news[r])
    assert torch.equal(k_pool.view(torch.int16), k0.view(torch.int16))      # the op does not write the pools
    assert torch.equal(v_pool.view(torch.int16), v0.view(torch.int16))
    again = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, max(news), slopes, D)
    assert torch.equal(out, again)
    # a loose bound on the new tokens changes the grid, not the result
    loose = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, table.shape[1] * PAGE_SIZE, slopes, D)
    assert torch.equal(out, loose)


@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_prefill_kernel_agrees_with_flash_kernel(D):
    """All starts 0: the same packed tokens through the document-masked flash kernel (keys from qkv) and through the
    paged kernel (keys stored into shuffled pages by paged_kv_write)."""
    H = 4
    news = [1, 127, 129, 1000, 64, 300]
    g = torch.Generator(device="cuda").manual_seed(D + 1)
    N = sum(news)
    qkv = torch.randn(N, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    need = [(n - 1) // PAGE_SIZE + 1 for n in news]
    perm = torch.randperm(sum(need) + 3, device="cuda", generator=g).to(torch.int32)
    table = torch.zeros(len(news), max(need), dtype=torch.int32, device="cuda")
    seg, slot, o, used = [], [], 0, 0
    for r, n in enumerate(news):
        table[r, :need[r]] = perm[used:used + need[r]]
        used += need[r]
        seg += [o] * n
        p = torch.arange(n, device="cuda")
        slot.append(table[r, p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE)
        o += n
    k_pool = torch.full((len(perm), H, PAGE_SIZE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    v_pool = k_pool.clone()
    paged_kv_write(qkv, torch.cat(slot).to(torch.int32), k_pool, v_pool, D)
    slopes = K.alibi_slopes(H, device="cuda")
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    start = torch.zeros(len(news), dtype=torch.int32, device="cuda")
    got = alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, max(news), slopes, D)
    seg = torch.tensor(seg, dtype=torch.int32, device="cuda").view(1, N)
    want = alibi_attention(qkv, slopes, 1, N, H, D, seg_start=seg)
    assert torch.isfinite(got).all()
    for r in range(len(news)):            # bf16 rounding: the two kernels block the keys differently
        rows = slice(int(cu[r]), int(cu[r + 1]))
        assert _rel(got[rows], want[rows]) < 1e-2, news[r]


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


def _check_cached_engine(model):
    """Requests that start with one of two shared system prompts, submitted in waves into a pool small enough that
    admissions wait and cached pages are evicted.  Every step's logits of each request against the training forward on
    its prompt + generated tokens; tokens against the arg-max wherever the top-2 margin exceeds twice the tolerance,
    and against generate() on the prompt alone until the first near-tie."""
    from pipegoose_b200.serving import ContinuousBatcher

    g = torch.Generator().manual_seed(11)
    systems = [torch.randint(0, 4096, (n,), generator=g).tolist() for n in (130, 200)]
    prompts, news = [], []
    for i in range(12):
        n = int(torch.randint(1, 120, (1,), generator=g))
        prompts.append(systems[i % 2] + torch.randint(0, 4096, (n,), generator=g).tolist())
        news.append(int(torch.randint(1, 24, (1,), generator=g)))
    engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE, max_prefill_tokens=400, prefix_caching=True)
    steps = {}
    forward = engine._forward

    def spy():
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps.setdefault(r.rid, []).append(logits[j].clone())
        return reqs, logits

    engine._forward = spy
    rids, outs = {}, {}
    for i in range(4):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(3):
        outs.update(engine.step())
    for i in range(4, 12):
        rids[i] = engine.submit(prompts[i], news[i])
        outs.update(engine.step())
    outs.update(engine.run())
    assert len(engine._free) == engine.num_pages
    assert engine.cached_prompt_tokens > 0
    for i, rid in rids.items():
        P, out = len(prompts[i]), outs[rid]
        assert len(out) == P + news[i] and len(steps[rid]) == news[i]
        with torch.no_grad():
            full = model(torch.tensor([out], device="cuda")).logits[0].float()
            alone = model.generate(torch.tensor([prompts[i]], device="cuda"), max_new_tokens=news[i])[0].tolist()
        tol = 3e-2 * full[P - 1:].abs().max().item()
        diverged = False
        for s, got in enumerate(steps[rid]):
            want = full[P - 1 + s]
            assert (got - want).abs().max().item() <= tol, (i, s, (got - want).abs().max().item(), tol)
            top2 = want.topk(2).values
            sure = bool(top2[0] - top2[1] > 2 * tol)
            if sure:
                assert out[P + s] == int(want.argmax()), (i, s)
            diverged = diverged or not sure
            if not diverged:
                assert out[P + s] == alone[P + s], (i, s)


@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_cached_engine_matches_training_forward(arch, hidden, n_head):
    _check_cached_engine((_bloom if arch == "bloom" else _gpt2)(hidden, n_head))


def test_cached_engine_with_expert_mlps():
    model, ctx = _moe_bloom()
    try:
        _check_cached_engine(model)
    finally:
        ctx.destroy()


def test_shared_pages_are_not_written():
    """The pages a request reuses hold the same bytes, in every layer, before and after it runs."""
    from pipegoose_b200.serving import ContinuousBatcher

    model = _bloom(320, 4)
    g = torch.Generator().manual_seed(12)
    system = torch.randint(0, 4096, (200,), generator=g).tolist()
    engine = ContinuousBatcher(model, max_cache_tokens=32 * PAGE_SIZE, prefix_caching=True)
    a = engine.submit(system + [5, 6], 40)
    engine.step()                                          # a's prompt: three full pages indexed
    shared = list(engine._admitted or engine._running)[0].pages[:3]
    snap_k, snap_v = engine.k_pools[:, shared].clone(), engine.v_pools[:, shared].clone()
    b = engine.submit(system + [7] * 90, 30)               # reuses the three pages while a decodes
    outs = engine.run()
    assert engine.cached_prompt_tokens == 3 * PAGE_SIZE
    assert torch.equal(engine.k_pools[:, shared].view(torch.int16), snap_k.view(torch.int16))
    assert torch.equal(engine.v_pools[:, shared].view(torch.int16), snap_v.view(torch.int16))
    assert sorted(outs) == [a, b]
