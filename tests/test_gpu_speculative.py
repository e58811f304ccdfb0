"""Speculative decoding on the GPU: the paged append-attention kernel against its fp32 reference (cached lengths from 0
to 33000, 1 to 8 appended tokens, NaN outside the valid slots, shuffled pages), its pool writes, its repeatability,
cross-checks against the paged prefill and paged decode kernels, and ``ContinuousBatcher(num_speculative_tokens=k)``
on bf16 Bloom at D = 64 and D = 80, and at D = 32, which has no kernel and verifies through the reference."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_paged_append_attention, alibi_paged_decode_attention,
                                          alibi_paged_prefill_attention, paged_kv_write)

pytestmark = pytest.mark.gpu

CACHED = [0, 1, 63, 64, 65, 1000, 4097, 33000]


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _case(H, D, starts, news, seed):
    """NaN pools with random keys / values in slots 0 .. starts[r] - 1 of every row only, a shuffled page table, and
    the appended tokens' qkv packed back to back."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(s + n - 1) // PAGE_SIZE + 1 for s, n in zip(starts, news)]
    num_pages = sum(need) + 3
    perm = torch.randperm(num_pages, device="cuda", generator=g).to(torch.int32)
    table = torch.full((len(starts), max(need) + 1), -7, dtype=torch.int32, device="cuda")   # never read
    k_pool = torch.full((num_pages, H, PAGE_SIZE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    v_pool = k_pool.clone()
    used = 0
    for r, s in enumerate(starts):
        table[r, :need[r]] = perm[used:used + need[r]]
        used += need[r]
        p = torch.arange(s, device="cuda")
        pages, slots = table[r, p // PAGE_SIZE].long(), p % PAGE_SIZE
        k_pool[pages, :, slots] = torch.randn(s, H, D, device="cuda", generator=g).to(torch.bfloat16)
        v_pool[pages, :, slots] = torch.randn(s, H, D, device="cuda", generator=g).to(torch.bfloat16)
    qkv = torch.randn(sum(news), H * 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    return qkv, k_pool, v_pool, table, cu, torch.tensor(starts, dtype=torch.int32, device="cuda")


def _slots(table, starts, news):
    return torch.tensor([int(table[r, p // PAGE_SIZE]) * PAGE_SIZE + p % PAGE_SIZE
                         for r, (s, n) in enumerate(zip(starts, news)) for p in range(s, s + n)], device="cuda")


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("most", [2, 3, 4, 8])                   # query tiles 2, 4, 4 and 8
@pytest.mark.parametrize("shift", [0, 3])
def test_append_kernel_matches_reference(D, most, shift):
    H = 2
    starts = CACHED
    news = [(i + shift) % most + 1 for i in range(len(starts))]    # 1 .. most tokens; rows 63 / 1000 ... cross pages
    qkv, k_pool, v_pool, table, cu, pos = _case(H, D, starts, news, seed=D + shift + 10 * most)
    slopes = K.alibi_slopes(H, device="cuda")
    max_pos = max(s + n - 1 for s, n in zip(starts, news))
    k0, v0 = k_pool.clone(), v_pool.clone()
    kf, vf = k_pool.float(), v_pool.float()
    ref = alibi_paged_append_attention(qkv.float(), kf, vf, table, cu.cpu(), pos.cpu(), max_pos, slopes, D)
    out = alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, max_pos, slopes, D, max_tokens=most)
    assert torch.isfinite(out).all()
    for r in range(len(starts)):
        rows = slice(int(cu[r]), int(cu[r + 1]))
        assert _rel(out[rows], ref[rows]) < 1e-2, (starts[r], news[r])

    # the new slots hold qkv's k / v bit for bit, and nothing else changed
    slot = _slots(table, starts, news)
    x = qkv.view(-1, H, 3, D)
    want_k, want_v = k0.clone(), v0.clone()
    want_k[slot // PAGE_SIZE, :, slot % PAGE_SIZE] = x[:, :, 1]
    want_v[slot // PAGE_SIZE, :, slot % PAGE_SIZE] = x[:, :, 2]
    assert torch.equal(k_pool.view(torch.int16), want_k.view(torch.int16))
    assert torch.equal(v_pool.view(torch.int16), want_v.view(torch.int16))

    # repeatable bit for bit; a loose max_pos (other splits) agrees within rounding
    again = alibi_paged_append_attention(qkv, k0.clone(), v0.clone(), table, cu, pos, max_pos, slopes, D,
                                         max_tokens=most)
    assert torch.equal(again.view(torch.int16), out.view(torch.int16))
    loose = alibi_paged_append_attention(qkv, k0.clone(), v0.clone(), table, cu, pos,
                                         table.shape[1] * PAGE_SIZE - 1, slopes, D, max_tokens=most)
    assert _rel(loose, out) < 1e-2
    wide = alibi_paged_append_attention(qkv, k0.clone(), v0.clone(), table, cu, pos, max_pos, slopes, D,
                                        max_tokens=8)                # the widest tile on the same rows
    assert _rel(wide, out) < 1e-2


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_append_kernel_single_row(D, n):
    """One row, its tile taken from host cu_seqlens (the smallest that holds n), against the reference."""
    H = 4
    qkv, k_pool, v_pool, table, cu, pos = _case(H, D, [4097 - n // 2], [n], seed=D + n)
    slopes = K.alibi_slopes(H, device="cuda")
    max_pos = 4096 + n
    ref = alibi_paged_append_attention(qkv.float(), k_pool.float(), v_pool.float(), table, cu.cpu(), pos.cpu(),
                                       max_pos, slopes, D)
    out = alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu.cpu(), pos.cpu(), max_pos, slopes, D)
    assert _rel(out, ref) < 1e-2


@pytest.mark.parametrize("D", [64, 80, 128])
def test_append_kernel_agrees_with_paged_prefill_and_decode(D):
    H = 4
    starts = [5, 64, 700, 2050]
    news = [8, 3, 5, 1]
    qkv, k_pool, v_pool, table, cu, pos = _case(H, D, starts, news, seed=7 * D)
    slopes = K.alibi_slopes(H, device="cuda")
    max_pos = max(s + n - 1 for s, n in zip(starts, news))
    kp, vp = k_pool.clone(), v_pool.clone()
    out = alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, max_pos, slopes, D, max_tokens=max(news))
    paged_kv_write(qkv, _slots(table, starts, news).to(torch.int32), kp, vp, D)
    pre = alibi_paged_prefill_attention(qkv, kp, vp, table, cu, pos, max(news), slopes, D)
    assert _rel(out, pre) < 1e-2

    news1 = [1] * len(starts)                                       # one token per row: the decode kernel's job
    qkv, k_pool, v_pool, table, cu, pos = _case(H, D, starts, news1, seed=11 * D)
    kd, vd = k_pool.clone(), v_pool.clone()
    out = alibi_paged_append_attention(qkv, k_pool, v_pool, table, cu, pos, max(starts), slopes, D, max_tokens=1)
    dec = alibi_paged_decode_attention(qkv, kd, vd, table, pos, max(starts), slopes, D)
    assert _rel(out, dec) < 1e-2
    assert torch.equal(k_pool.view(torch.int16), kd.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------ engine
def _bloom(hidden):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(0)
    cfg = BloomConfig(vocab_size=256, hidden_size=hidden, n_layer=2, n_head=4, initializer_range=0.2)
    with torch.device("cuda"):
        return BloomForCausalLM(cfg).to(torch.bfloat16).eval()


def _prompts(n, seed=0, vocab=256):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        base = torch.randint(0, vocab, (int(torch.randint(4, 12, (1,), generator=g)),), generator=g).tolist()
        out.append((base * 8)[:20 + 9 * i] + torch.randint(0, vocab, (5,), generator=g).tolist())
    return out


@pytest.mark.parametrize("hidden", [256, 320, 128])   # D = 64, 80, and 32 (no kernel: the reference path)
def test_engine_greedy_matches_full_forward_argmax(hidden):
    from pipegoose_b200.serving import ContinuousBatcher

    model = _bloom(hidden)
    prompts = _prompts(8)
    eng = ContinuousBatcher(model, max_cache_tokens=64 * 64, num_speculative_tokens=5)
    rids = [eng.submit(p, max_new_tokens=24 + 4 * i) for i, p in enumerate(prompts)]
    outs = eng.run()
    assert eng.speculative_accepted_tokens > 0
    with torch.no_grad():
        for r, prompt in zip(rids, prompts):
            toks = outs[r]
            logits = model(torch.tensor(toks[:-1], device="cuda").view(1, -1)).logits[0].float()
            for t in range(len(prompt) - 1, len(toks) - 1):
                top2 = logits[t].topk(2).values
                if toks[t + 1] != int(logits[t].argmax()):     # bf16 rounding: only near-ties may differ
                    assert float(top2[0] - top2[1]) < 3e-2 * max(1.0, float(top2[0].abs())), (t, toks[t + 1])
    assert len(eng._free) == eng.num_pages


@pytest.mark.parametrize("hidden", [256, 320])
def test_engine_without_drafts_is_the_decode_path(hidden, monkeypatch):
    from pipegoose_b200 import serving

    model = _bloom(hidden)
    prompts = _prompts(6, seed=1)
    plain = serving.ContinuousBatcher(model, max_cache_tokens=64 * 64)
    rp = [plain.submit(p, max_new_tokens=20) for p in prompts]
    want = plain.run()
    monkeypatch.setattr(serving._NgramIndex, "draft", lambda self, tokens, k: [])
    spec = serving.ContinuousBatcher(model, max_cache_tokens=64 * 64, num_speculative_tokens=7)
    rs = [spec.submit(p, max_new_tokens=20) for p in prompts]
    got = spec.run()
    assert [got[r] for r in rs] == [want[r] for r in rp]
    assert spec.speculative_proposed_tokens == 0
