"""The decode-attention reference (ops/attention.py) against the attention math of the eager KV-cached path in
models/bloom.py: a cache grown by ``cat``, fp32 scores with ``slope * key_position``, the causal mask and pad keys masked
with the most negative finite value."""
import math

import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import alibi_decode_attention, alibi_decode_attention_reference


def _eager_step(q, k_prev, v_prev, k_new, v_new, slopes, lead):
    """models/bloom.py's eager attention for one new position (T = 1); ``q``, ``k_new``, ``v_new``: [B, H, 1, D]."""
    k = torch.cat([k_prev, k_new], dim=2)
    v = torch.cat([v_prev, v_new], dim=2)
    S, D, H = k.shape[2], k.shape[3], k.shape[1]
    past = S - 1
    scores = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(D)
    key_pos = torch.arange(S, dtype=torch.float32)
    scores = scores + slopes.view(1, H, 1, 1) * key_pos
    scores = scores.masked_fill(key_pos.view(1, S) > torch.arange(past, past + 1).view(1, 1), float("-inf"))
    if lead is not None:
        pad = key_pos.view(1, 1, 1, -1) < lead.view(-1, 1, 1, 1).to(key_pos.dtype)
        scores = scores.masked_fill(pad, torch.finfo(scores.dtype).min)
    return torch.matmul(scores.softmax(-1).to(v.dtype), v)            # [B, H, 1, D]


def _case(B, H, D, pos, capacity, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, H * 3 * D, generator=g).to(dtype)
    k_cache = torch.randn(B, H, capacity, D, generator=g).to(dtype)
    v_cache = torch.randn(B, H, capacity, D, generator=g).to(dtype)
    return qkv, k_cache, v_cache


@pytest.mark.parametrize("D", [64, 80, 128])
@pytest.mark.parametrize("alibi", [True, False])
@pytest.mark.parametrize("with_lead", [False, True])
def test_reference_matches_the_eager_cached_attention(D, alibi, with_lead):
    B, H, pos, capacity = 3, 4, 37, 50
    qkv, k_cache, v_cache = _case(B, H, D, pos, capacity, seed=D)
    slopes = K.alibi_slopes(H) if alibi else torch.zeros(H)
    lead = torch.tensor([0, 5, pos]) if with_lead else None     # the last row sees exactly one key
    x = qkv.view(B, H, 3, D)
    want = _eager_step(x[:, :, 0:1], k_cache[:, :, :pos], v_cache[:, :, :pos], x[:, :, 1:2], x[:, :, 2:3], slopes, lead)
    got = alibi_decode_attention_reference(qkv, k_cache, v_cache, slopes, pos, lead, D)
    torch.testing.assert_close(got, want.reshape(B, H * D), rtol=1e-5, atol=1e-5)
    if with_lead:       # one visible key: the output is that key's value, the new v
        torch.testing.assert_close(got.view(B, H, D)[2], x[2, :, 2], rtol=1e-6, atol=1e-6)


def test_cache_write_touches_only_pos():
    B, H, D, pos, capacity = 2, 3, 64, 9, 16
    qkv, k_cache, v_cache = _case(B, H, D, pos, capacity, dtype=torch.bfloat16, seed=1)
    k0, v0 = k_cache.clone(), v_cache.clone()
    alibi_decode_attention(qkv, k_cache, v_cache, K.alibi_slopes(H), pos, torch.tensor([0, 3]), D)
    x = qkv.view(B, H, 3, D)
    assert torch.equal(k_cache[:, :, pos], x[:, :, 1]) and torch.equal(v_cache[:, :, pos], x[:, :, 2])
    keep = torch.ones(capacity, dtype=torch.bool)
    keep[pos] = False
    assert torch.equal(k_cache[:, :, keep], k0[:, :, keep]) and torch.equal(v_cache[:, :, keep], v0[:, :, keep])


def test_cpu_tensors_dispatch_to_the_reference():
    B, H, D, pos, capacity = 2, 2, 80, 6, 8
    qkv, k_cache, v_cache = _case(B, H, D, pos, capacity, dtype=torch.bfloat16, seed=2)
    slopes = K.alibi_slopes(H)
    k_ref, v_ref = k_cache.clone(), v_cache.clone()
    want = alibi_decode_attention_reference(qkv, k_ref, v_ref, slopes, pos, None, D)
    got = alibi_decode_attention(qkv, k_cache, v_cache, slopes, pos, None, D)
    assert torch.equal(got, want) and torch.equal(k_cache, k_ref) and torch.equal(v_cache, v_ref)


def test_position_outside_the_capacity_is_refused():
    qkv, k_cache, v_cache = _case(1, 2, 64, 4, 4)
    with pytest.raises(ValueError, match="capacity"):
        alibi_decode_attention(qkv, k_cache, v_cache, torch.zeros(2), 4, None, 64)
