"""KV-cached decoding on the GPU: the split-KV decode kernel against the fp32 reference, the flash-kernel prefill of
left-padded prompts, native generate() against full recomputation (Bloom, GPT-2, head sizes 64 / 80 / 128, expert
MLPs), linear memory in the prompt length, and tensor parallelism."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


# filled lengths (pos + 1): one split, split-chunk boundaries, many splits
LENGTHS = [1, 2, 63, 64, 65, 1000, 4097, 33000]


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("filled", LENGTHS)
def test_decode_kernel_matches_reference(D, filled):
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_decode_attention, alibi_decode_attention_reference

    pos = filled - 1
    for B, H, lead in ((1, 2, None), (3, 4, [0, pos // 2, pos])):
        g = torch.Generator(device="cuda").manual_seed(filled * 7 + D)
        cap = filled + 3
        qkv = torch.randn(B, H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
        k_cache = torch.randn(B, H, cap, D, device="cuda", generator=g).to(torch.bfloat16)
        v_cache = torch.randn(B, H, cap, D, device="cuda", generator=g).to(torch.bfloat16)
        slopes = K.alibi_slopes(H, device="cuda")
        lead_t = None if lead is None else torch.tensor(lead, device="cuda", dtype=torch.int32)
        k0, v0 = k_cache.clone(), v_cache.clone()
        out = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, lead_t, D)
        ref = alibi_decode_attention_reference(qkv.float(), k0.float(), v0.float(), slopes, pos, lead_t, D)
        assert torch.isfinite(out).all()
        assert _rel(out, ref) < 1e-2, (B, H)
        x = qkv.view(B, H, 3, D)
        assert torch.equal(k_cache[:, :, pos], x[:, :, 1]) and torch.equal(v_cache[:, :, pos], x[:, :, 2])
        keep = torch.ones(cap, dtype=torch.bool, device="cuda")
        keep[pos] = False
        assert torch.equal(k_cache[:, :, keep], k0[:, :, keep]) and torch.equal(v_cache[:, :, keep], v0[:, :, keep])
        again = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, lead_t, D)
        assert torch.equal(out, again)
        if lead is not None:     # the row with lead == pos sees only the new key: its output is the new value
            assert torch.equal(out.view(B, H, D)[2], x[2, :, 2])


def test_decode_kernel_refuses_bad_arguments():
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_decode_attention

    B, H, D, cap = 2, 2, 96, 8
    qkv = torch.zeros(B, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    cache = torch.zeros(B, H, cap, D, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="head size"):
        alibi_decode_attention(qkv, cache, cache.clone(), K.alibi_slopes(H, device="cuda"), 3, None, D)
    D = 64
    qkv = torch.zeros(B, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    cache = torch.zeros(B, H, cap, D, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="capacity"):
        alibi_decode_attention(qkv, cache, cache.clone(), K.alibi_slopes(H, device="cuda"), cap, None, D)


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
    from pipegoose_b200.nn import ExpertParallel
    from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer
    from pipegoose_b200.nn.expert_parallel.routers import Top2Router
    from pipegoose_b200.testing.utils import find_free_port, init_parallel_context

    ctx = init_parallel_context(0, 1, find_free_port(), 1, 1, 1, backend="nccl")
    torch.manual_seed(0)
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=256, n_layer=2, n_head=4))
    model = ExpertParallel(model, 4, mapping=[1], router=Top2Router(None, 4, 256), parallel_context=ctx,
                           fused=False).parallelize()
    assert type(model.transformer.h[1].mlp) is ExpertLayer
    return model.to(torch.bfloat16).cuda().eval(), ctx


def test_left_padded_prefill_matches_rows_run_alone():
    model = _bloom(256, 4)
    lengths = [37, 200, 129]
    P = max(lengths)
    ids = torch.randint(0, 4096, (len(lengths), P), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    lead = torch.tensor([P - n for n in lengths], device="cuda")
    with torch.no_grad():
        cache = [None] * 2
        batch = model._incremental_logits(ids, cache, 0, lead, capacity=P + 4)[:, -1].float()
        assert all(c[0].shape[2] == P and c[2].shape[2] == P + 4 for c in cache)
        for b, n in enumerate(lengths):
            alone = model._incremental_logits(ids[b:b + 1, P - n:], [None] * 2, 0)[:, -1].float()
            assert _rel(batch[b], alone[0]) < 2e-2, b


def _check_generate(model, ids, attention_mask=None, new=12):
    """Per-step logits of the cached (native) path against the training forward on the same tokens; greedy tokens
    against use_cache=False wherever the top-2 margin exceeds the bf16 tolerance."""
    B, P = ids.shape
    out = model.generate(ids, max_new_tokens=new, attention_mask=attention_mask)
    lead = None if attention_mask is None else (attention_mask.cumsum(1) == 0).sum(1)
    full_mask = None if attention_mask is None else torch.cat([attention_mask, attention_mask.new_ones(B, new)], 1)
    with torch.no_grad():
        full = (model(out, attention_mask=full_mask) if full_mask is not None else model(out)).logits.float()
        cache = [None] * len(model.transformer.h)
        steps = [model._incremental_logits(out[:, :P], cache, 0, lead, capacity=P + new)[:, -1].float()]
        for i in range(1, new):
            steps.append(model._incremental_logits(out[:, P + i - 1:P + i], cache, P + i - 1, lead)[:, -1].float())
    assert cache[0][0].shape[2] == P + new - 1 and cache[0][2].shape[2] == P + new
    ref = model.generate(ids, max_new_tokens=new, attention_mask=attention_mask, use_cache=False)
    tol = 3e-2 * full[:, P - 1:].abs().max().item()
    diverged = False
    for i, step in enumerate(steps):
        want = full[:, P - 1 + i]
        assert (step - want).abs().max().item() <= tol, (i, (step - want).abs().max().item(), tol)
        top2 = want.topk(2, dim=-1).values
        sure = (top2[:, 0] - top2[:, 1]) > 2 * tol
        assert torch.equal(out[:, P + i][sure], want.argmax(-1)[sure]), i
        diverged = diverged or not bool(sure.all())
        if not diverged:
            assert torch.equal(out[:, P + i], ref[:, P + i]), i


@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("gpt2", 256, 4), ("bloom", 320, 4),
                                                  ("bloom", 512, 4)])
@pytest.mark.parametrize("padded", [False, True])
def test_generate_matches_full_recomputation(arch, hidden, n_head, padded):
    model = (_bloom if arch == "bloom" else _gpt2)(hidden, n_head)
    g = torch.Generator("cuda").manual_seed(11)
    ids = torch.randint(0, 4096, (3, 70), device="cuda", generator=g)
    mask = None
    if padded:
        mask = torch.ones_like(ids)
        mask[0, :13] = 0
        mask[2, :69] = 0        # a one-token prompt
    _check_generate(model, ids, mask)


def test_generate_with_expert_mlps():
    model, ctx = _moe_bloom()
    try:
        ids = torch.randint(0, 4096, (2, 40), device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        _check_generate(model, ids, new=8)
    finally:
        ctx.destroy()


def test_prefill_memory_is_linear_in_the_prompt():
    model = _bloom(256, 4, vocab=4096)
    B, T, H, D, h, L, new = 2, 16384, 4, 64, 256, 2, 4
    ids = torch.randint(0, 4096, (B, T), device="cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = model.generate(ids, max_new_tokens=new)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    assert out.shape == (B, T + new)
    cache = 2 * L * B * H * (T + new) * D * 2                 # bf16 k and v of every layer
    widest = B * T * 4 * h * 2                                  # the MLP's bf16 [tokens, 4h] activation
    bound = cache + 8 * widest
    eager_scores = B * H * T * T * 4                            # the eager path's fp32 [B, H, T, T] scores of one layer
    assert bound * 10 < eager_scores
    assert rise < bound, (rise, bound)


def run_tp_generate(rank, world_size, port, state, ids, ref_tokens):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.nn import TensorParallel
    from pipegoose_b200.testing.utils import init_parallel_context

    ctx = init_parallel_context(rank, world_size, port, world_size, 1, 1, backend="nccl")
    model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=256, n_layer=2, n_head=4))
    model.load_state_dict(state)
    model = TensorParallel(model.to(torch.bfloat16), ctx).parallelize()
    model.to("cuda").eval()
    out = model.generate(ids.cuda(), max_new_tokens=ref_tokens.shape[1] - ids.shape[1])
    assert torch.equal(out.cpu(), ref_tokens)
    ctx.destroy()


def test_tp2_generate_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pipegoose_b200.testing.utils import spawn

    model = _bloom(256, 4)
    state = copy.deepcopy({k: v.float().cpu() for k, v in model.state_dict().items()})
    ids = torch.randint(0, 4096, (2, 64), generator=torch.Generator().manual_seed(2))
    ref = model.generate(ids.cuda(), max_new_tokens=8).cpu()
    spawn(run_tp_generate, world_size=2, state=state, ids=ids, ref_tokens=ref)
