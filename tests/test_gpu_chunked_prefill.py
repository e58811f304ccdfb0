"""Chunked prefill on the GPU: the FP8 form of the paged prefill kernel bit for bit against the staged path (the bf16
kernel over dequantized pages) and against the fp32 reference, and ``ContinuousBatcher(chunked_prefill=True)`` against
the training forward (teacher-forced), with bf16 and FP8 pools."""
import pytest
import torch

from pipegoose_b200.ops import attention as A
from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_paged_prefill_attention,
                                          alibi_paged_prefill_attention_reference, fp8_prefill_staging, quantize_kv)

pytestmark = pytest.mark.gpu

FP8 = torch.float8_e4m3fn


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-6)


def _fp8_case(H, D, starts, news, seed, spare_pages=5):
    """Pools of NaN codes and NaN scales with quantized random keys / values in every sequence's cached positions
    ``0 .. starts[r] - 1``, shuffled page tables, and ``qkv`` of the new tokens; all on the CPU."""
    g = torch.Generator().manual_seed(seed)
    lengths = [s + n for s, n in zip(starts, news)]
    need = [(n - 1) // PAGE_SIZE + 1 for n in lengths]
    num_pages = sum(need) + spare_pages
    perm = torch.randperm(num_pages, generator=g).to(torch.int32)
    table = torch.full((len(lengths), max(need) + 1), -7, dtype=torch.int32)   # never read
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), 0x7F, dtype=torch.uint8).view(FP8)
    scales = torch.full((num_pages, H, PAGE_SIZE), float("nan"))
    v_pool, k_scales, v_scales = k_pool.clone(), scales, scales.clone()
    used = 0
    for r, s in enumerate(starts):
        table[r, :need[r]] = perm[used:used + need[r]]
        used += need[r]
        p = torch.arange(s)
        pages, slots = table[r, p // PAGE_SIZE].long(), p % PAGE_SIZE
        for pool, sc in ((k_pool, k_scales), (v_pool, v_scales)):
            codes, x = quantize_kv(torch.randn(s, H, D, generator=g).to(torch.bfloat16))
            pool[pages, :, slots], sc[pages, :, slots] = codes, x
    qkv = torch.randn(sum(news), H * 3 * D, generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32)
    return k_pool, v_pool, k_scales, v_scales, table, qkv, cu, lengths


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("starts,news", [([0, 64, 192, 8192], [129, 1, 1000, 300]),
                                         ([8192, 0, 640, 64, 128], [64, 127, 128, 513, 1])])
def test_fp8_prefill_kernel_is_bitwise_the_staged_path(D, starts, news):
    """Several sequences on shuffled pages, cached prefixes of 0, 1, an odd number of pages and 8192 positions, pool
    slots past each sequence's cached positions holding NaN codes and NaN scales.  The FP8 kernel's output equals the
    bf16 kernel's over the staging pool bit for bit, and the fp32 reference within the prefill tests' tolerance."""
    H = 3
    k_pool, v_pool, k_scales, v_scales, table, qkv, cu, lengths = _fp8_case(H, D, starts, news, seed=D + len(starts))
    slopes = K.alibi_slopes(H, device="cuda")
    gpu = [t.cuda() for t in (k_pool, v_pool, k_scales, v_scales)]
    start = torch.tensor(starts, dtype=torch.int32)
    args = (qkv.cuda(), gpu[0], gpu[1], table.cuda(), cu.cuda(), start.cuda(), max(news), slopes, D)
    got = alibi_paged_prefill_attention(*args, k_scales=gpu[2], v_scales=gpu[3])
    pages = [table[r, :(n - 1) // PAGE_SIZE + 1].tolist() for r, n in enumerate(lengths)]
    n, src, dst, slot, st_table = fp8_prefill_staging(pages, starts, lengths)
    k_stage = torch.full((n, H, PAGE_SIZE, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    dev = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
    stage = (k_stage, k_stage.clone(), dev(src), dev(dst), dev(slot), dev(st_table))
    staged = alibi_paged_prefill_attention(*args, k_scales=gpu[2], v_scales=gpu[3], stage=stage)
    assert torch.isfinite(got).all()
    assert torch.equal(got.view(torch.int16), staged.view(torch.int16))
    want = alibi_paged_prefill_attention_reference(qkv.float(), k_pool, v_pool, table, cu, start, max(news),
                                                   slopes.cpu(), D, k_scales=k_scales, v_scales=v_scales)
    for r in range(len(starts)):
        assert _rel(got[cu[r]:cu[r + 1]], want[cu[r]:cu[r + 1]]) < 1e-2, (starts[r], news[r])
    for before, after in zip((k_pool, v_pool), gpu):                      # the op does not write the pools
        assert torch.equal(before.view(torch.uint8), after.cpu().view(torch.uint8))


def test_fp8_prefill_kernel_refusals():
    H, D = 2, 64
    k_pool, v_pool, k_scales, v_scales, table, qkv, cu, _ = _fp8_case(H, D, [64], [10], seed=1)
    slopes = K.alibi_slopes(H, device="cuda")
    gpu = [t.cuda() for t in (k_pool, v_pool, k_scales, v_scales, qkv)]
    with pytest.raises(ValueError, match="multiple of 64"):
        alibi_paged_prefill_attention(gpu[4], gpu[0], gpu[1], table.cuda(), cu, torch.tensor([32], dtype=torch.int32),
                                      10, slopes, D, k_scales=gpu[2], v_scales=gpu[3])
    with pytest.raises(RuntimeError, match="bf16"):
        A.native().paged_prefill_attention_fp8(gpu[4].float(), gpu[0], gpu[1], gpu[2], gpu[3], table.cuda(),
                                               cu.cuda(), torch.tensor([64], dtype=torch.int32, device="cuda"), 10,
                                               slopes, torch.empty(10, H * D, device="cuda", dtype=torch.bfloat16),
                                               0.0)


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


@pytest.mark.parametrize("chunked", [False, True])
def test_fp8_kernel_is_bitwise_the_staged_path_on_engine_inputs(monkeypatch, chunked):
    """Every cached-prefix prefill call of the FP8 engine (prefix hits; with chunking, every chunk) gives the same bits
    through the FP8 kernel as through the staged path."""
    from pipegoose_b200.serving import ContinuousBatcher

    model = _model("bloom", 320, 4)
    prompts, news = _workload(seed=17)
    op, calls = A.alibi_paged_prefill_attention, [0]

    def both(qkv, k_pool, v_pool, table, cu_seqlens, start, max_len, slopes, D, softmax_scale=0.0, k_scales=None,
             v_scales=None, stage=None, out=None):
        got = op(qkv, k_pool, v_pool, table, cu_seqlens, start, max_len, slopes, D, k_scales=k_scales,
                 v_scales=v_scales)
        if k_scales is not None:
            cu, st, tb = cu_seqlens.tolist(), start.tolist(), table.tolist()
            lengths = [s + cu[r + 1] - cu[r] for r, s in enumerate(st)]
            pages = [tb[r][:(n - 1) // PAGE_SIZE + 1] for r, n in enumerate(lengths)]
            n, src, dst, slot, st_table = fp8_prefill_staging(pages, st, lengths)
            k_stage = torch.empty(n, k_pool.shape[1], PAGE_SIZE, D, dtype=torch.bfloat16, device="cuda")
            dev = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
            stage = (k_stage, torch.empty_like(k_stage), dev(src), dev(dst), dev(slot), dev(st_table))
            staged = op(qkv, k_pool, v_pool, table, cu_seqlens, start, max_len, slopes, D, k_scales=k_scales,
                        v_scales=v_scales, stage=stage)
            assert torch.equal(got.view(torch.int16), staged.view(torch.int16))
            calls[0] += 1
        return got if out is None else out.copy_(got)
    monkeypatch.setattr(A, "alibi_paged_prefill_attention", both)
    engine = ContinuousBatcher(model, max_cache_tokens=24 * PAGE_SIZE, max_prefill_tokens=128 if chunked else 400,
                               prefix_caching=True, kv_cache_dtype=FP8, chunked_prefill=chunked)
    for p, n in zip(prompts, news):
        engine.submit(p, n)
    engine.run()
    assert engine.cached_prompt_tokens > 0 and calls[0] > 0
