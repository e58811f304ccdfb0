"""Continuous batching on the GPU: the paged form of the split-KV decode kernel against its fp32 reference (rows of
different lengths, shuffled page tables, NaN outside the valid slots), its agreement with the contiguous kernel, the
prefill cache write, and ``ContinuousBatcher`` on bf16 models against the training forward and ``generate()``."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_decode_attention, alibi_paged_decode_attention,
                                          alibi_paged_decode_attention_reference, paged_kv_write,
                                          paged_kv_write_reference)

pytestmark = pytest.mark.gpu

LENGTHS = [1, 2, 63, 64, 65, 1000, 4097, 33000]


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _bits(t):
    return t.view(torch.int16)


def _paged_case(H, D, lengths, spare_pages, seed):
    """NaN pools with random keys / values in every row's slots before its position, and a shuffled page table."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(n - 1) // PAGE_SIZE + 1 for n in lengths]
    num_pages = sum(need) + spare_pages
    perm = torch.randperm(num_pages, device="cuda", generator=g).to(torch.int32)
    width = max(need) + 1
    table = torch.full((len(lengths), width), -7, dtype=torch.int32, device="cuda")   # never read
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    v_pool = k_pool.clone()
    used = 0
    for b, n in enumerate(lengths):
        table[b, :need[b]] = perm[used:used + need[b]]
        used += need[b]
        p = torch.arange(n - 1, device="cuda")         # the slots before the new position
        pages, slots = table[b, p // PAGE_SIZE].long(), p % PAGE_SIZE
        k_pool[pages, :, slots] = torch.randn(n - 1, H, D, device="cuda", generator=g).to(torch.bfloat16)
        v_pool[pages, :, slots] = torch.randn(n - 1, H, D, device="cuda", generator=g).to(torch.bfloat16)
    qkv = torch.randn(len(lengths), H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32, device="cuda")
    return qkv, k_pool, v_pool, table, pos


@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_kernel_matches_reference(D):
    H = 2
    lengths = LENGTHS[D % 3:] + LENGTHS[:D % 3]        # a different row order per head size
    qkv, k_pool, v_pool, table, pos = _paged_case(H, D, lengths, spare_pages=5, seed=D)
    slopes = K.alibi_slopes(H, device="cuda")
    max_pos = max(lengths) - 1
    k0, v0 = k_pool.clone(), v_pool.clone()
    out = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, max_pos, slopes, D)
    ref = alibi_paged_decode_attention_reference(qkv.float(), k0.float(), v0.float(), table, pos, max_pos, slopes, D)
    assert torch.isfinite(out).all()
    for b in range(len(lengths)):
        assert _rel(out[b], ref[b]) < 1e-2, lengths[b]
    # only the slot of pos[b] changed, and it holds the qkv row's k / v bit for bit
    x = qkv.view(-1, H, 3, D)
    for b, n in enumerate(lengths):
        page, off = table[b, (n - 1) // PAGE_SIZE].long(), (n - 1) % PAGE_SIZE
        assert torch.equal(k_pool[page, :, off], x[b, :, 1]) and torch.equal(v_pool[page, :, off], x[b, :, 2])
        k0[page, :, off], v0[page, :, off] = x[b, :, 1], x[b, :, 2]
    assert torch.equal(_bits(k_pool), _bits(k0)) and torch.equal(_bits(v_pool), _bits(v0))
    again = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, max_pos, slopes, D)
    assert torch.equal(out, again)
    # a loose bound on the positions changes the grid, not the result beyond rounding
    loose = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, table.shape[1] * PAGE_SIZE - 1, slopes, D)
    assert torch.isfinite(loose).all() and _rel(loose, ref) < 1e-2


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("pos", [0, 100, 5000])
def test_paged_kernel_equals_contiguous_kernel(D, pos):
    B, H = 3, 4
    cap = pos + 1
    g = torch.Generator(device="cuda").manual_seed(pos + D)
    qkv = torch.randn(B, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    n_pages = (cap - 1) // PAGE_SIZE + 1
    k_cache = torch.randn(B, H, n_pages * PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
    v_cache = torch.randn(B, H, n_pages * PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
    table = torch.randperm(B * n_pages, device="cuda", generator=g).to(torch.int32).view(B, n_pages)
    k_pool = torch.empty(B * n_pages, H, PAGE_SIZE, D, device="cuda", dtype=torch.bfloat16)
    v_pool = torch.empty_like(k_pool)
    pages = k_cache.view(B, H, n_pages, PAGE_SIZE, D).transpose(1, 2)       # [B, pages, H, 64, D]
    k_pool[table.long()] = pages
    v_pool[table.long()] = v_cache.view(B, H, n_pages, PAGE_SIZE, D).transpose(1, 2)
    slopes = K.alibi_slopes(H, device="cuda")
    want = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, None, D)
    pos_t = torch.full((B,), pos, dtype=torch.int32, device="cuda")
    got = alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos_t, pos, slopes, D)
    assert torch.equal(got, want)
    back_k = k_pool[table.long()].transpose(1, 2).reshape(B, H, -1, D)
    back_v = v_pool[table.long()].transpose(1, 2).reshape(B, H, -1, D)
    assert torch.equal(back_k, k_cache) and torch.equal(back_v, v_cache)


@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_kv_write_is_exact(D):
    N, H, num_pages = 777, 3, 20
    g = torch.Generator(device="cuda").manual_seed(D)
    qkv = torch.randn(N, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    slot = torch.randperm(num_pages * PAGE_SIZE, device="cuda", generator=g)[:N].to(torch.int32)
    k_pool = torch.randn(num_pages, H, PAGE_SIZE, D, device="cuda", generator=g).to(torch.bfloat16)
    v_pool = torch.randn_like(k_pool)
    k_ref, v_ref = k_pool.clone(), v_pool.clone()
    paged_kv_write(qkv, slot, k_pool, v_pool, D)
    paged_kv_write_reference(qkv, slot, k_ref, v_ref, D)
    assert torch.equal(k_pool, k_ref) and torch.equal(v_pool, v_ref)


def test_paged_ops_refuse_bad_arguments():
    H, D = 2, 64
    qkv = torch.zeros(1, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    pool = torch.zeros(2, H, 32, D, device="cuda", dtype=torch.bfloat16)         # pages of 32 positions
    table = torch.zeros(1, 1, dtype=torch.int32, device="cuda")
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    slopes = K.alibi_slopes(H, device="cuda")
    with pytest.raises(RuntimeError, match="page dimension"):
        alibi_paged_decode_attention(qkv, pool, pool.clone(), table, pos, 0, slopes, D)
    with pytest.raises(RuntimeError, match="page dimension"):
        paged_kv_write(qkv, pos, pool, pool.clone(), D)
    qkv96 = torch.zeros(1, H * 3 * 96, device="cuda", dtype=torch.bfloat16)
    pool96 = torch.zeros(2, H, PAGE_SIZE, 96, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="head size"):
        alibi_paged_decode_attention(qkv96, pool96, pool96.clone(), table, pos, 0, slopes, 96)


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


def _check_engine(model):
    """Staggered submissions into a pool small enough that admissions wait and pages are reused.  Every step's logits
    of each request against the training forward on its prompt + generated tokens; tokens against the arg-max wherever
    the top-2 margin exceeds twice the tolerance, and against generate() on the prompt alone until the first near-tie."""
    from pipegoose_b200.serving import ContinuousBatcher

    g = torch.Generator().manual_seed(7)
    lengths = [int(n) for n in torch.randint(1, 200, (12,), generator=g)]
    lengths[3] = 1
    news = [int(n) for n in torch.randint(1, 24, (12,), generator=g)]
    news[5] = 1
    prompts = [torch.randint(0, 4096, (n,), generator=g).tolist() for n in lengths]
    engine = ContinuousBatcher(model, max_cache_tokens=10 * PAGE_SIZE, max_prefill_tokens=300)
    steps = {}
    forward = engine._forward

    def spy():
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps.setdefault(r.rid, []).append(logits[j].clone())
        return reqs, logits

    engine._forward = spy
    rids, outs = {}, {}
    for i in range(6):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(4):
        outs.update(engine.step())
    for i in range(6, 12):
        rids[i] = engine.submit(prompts[i], news[i])
        outs.update(engine.step())
    outs.update(engine.run())
    assert len(engine._free) == engine.num_pages
    for i, rid in rids.items():
        P, out = lengths[i], outs[rid]
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
def test_engine_matches_training_forward(arch, hidden, n_head):
    _check_engine((_bloom if arch == "bloom" else _gpt2)(hidden, n_head))


def test_engine_with_expert_mlps():
    model, ctx = _moe_bloom()
    try:
        _check_engine(model)
    finally:
        ctx.destroy()
