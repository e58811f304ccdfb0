"""Causal ALiBi self-attention on Bloom's fused QKV layout.

``qkv`` is ``[B*S, n_head*3*D]`` with each row laid out ``[head][q|k|v][D]`` (the layout HF Bloom's
``query_key_value`` produces), the result is ``[B*S, n_head*D]``.  Scores are
``q.k / sqrt(D) + slope[head] * key_position`` under a causal mask, softmax in fp32.

Two implementations share this contract: the sm_90a flash kernel (``csrc/attention_sm90.cu``:
wgmma QK^T / PV with register accumulators, online softmax, never materialising ``[S, S]``) and
the PyTorch reference below (CPU tests, numerics oracle).

Packed sequences: ``seg_start`` (int32 ``[B, S]`` or ``[B*S]``, see :func:`seg_start_from_position_ids`) holds, for
every token, the row-relative position where its document begins.  Query ``q`` then sees key ``k`` iff
``seg_start[q] <= k <= q``: documents packed into one row do not attend to each other.  ``None``: one document per row.
"""
from __future__ import annotations

import math
from typing import Tuple

import torch

from pipegoose_b200.ops import has_kernel, native, use_native


def seg_start_from_position_ids(position_ids: torch.Tensor) -> torch.Tensor:
    """int32 ``[B, S]`` document starts of packed rows: ``seg_start[b, s] = s - position_ids[b, s]``, where every row of
    ``position_ids`` is a concatenation of runs ``0, 1, 2, ...`` (one per document).  Nothing is checked here; the models
    validate ``position_ids`` on the device first."""
    S = position_ids.shape[-1]
    pos = torch.arange(S, device=position_ids.device, dtype=position_ids.dtype)
    return (pos - position_ids).to(torch.int32).contiguous()


def visible_mask(S: int, device, seg_start=None, B: int = 1) -> torch.Tensor:
    """Boolean visibility of key ``k`` from query ``q``: ``[S, S]`` causal, or ``[B, 1, S, S]`` with the document lower
    bound ``k >= seg_start[b, q]`` of packed rows."""
    causal = torch.ones(S, S, dtype=torch.bool, device=device).tril()
    if seg_start is None:
        return causal
    k = torch.arange(S, device=device)
    return causal & (k.view(1, 1, 1, S) >= seg_start.reshape(B, 1, S, 1).to(device))


def alibi_attention_reference(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                              softmax_scale: float = 0.0, dropout_p: float = 0.0, seg_start=None) -> torch.Tensor:
    """``dropout_p > 0``: dropout on the attention probabilities (🤗 Bloom's ``attention_dropout``: zeroed entries, the
    rest scaled by ``1 / (1 - p)``, rows not re-normalised).  ``seg_start``: packed documents (module docstring)."""
    x = qkv.view(B, S, n_head, 3, D)
    q, k, v = (x[:, :, :, i].permute(0, 2, 1, 3).float() for i in range(3))  # [B, H, S, D]
    scores = torch.matmul(q, k.transpose(-1, -2)) * (softmax_scale if softmax_scale > 0 else 1.0 / math.sqrt(D))
    pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
    scores = scores + slopes.float().view(1, n_head, 1, 1) * pos.view(1, 1, 1, S)
    scores = scores.masked_fill(~visible_mask(S, qkv.device, seg_start, B), float("-inf"))
    p = torch.softmax(scores, dim=-1)
    if dropout_p > 0.0:
        p = torch.nn.functional.dropout(p, dropout_p, True)
    out = torch.matmul(p, v)  # [B, H, S, D]
    return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D).to(qkv.dtype)


def alibi_attention_with_dropout(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                                 dropout_p: float, seg_start=None) -> torch.Tensor:
    """Training-time attention with dropout on the probabilities.  The flash kernel never holds a row of probabilities
    (online softmax), so this path materialises them: bf16 GEMMs around an fp32 softmax, one head group at a time so
    that the live ``[B, heads, S, S]`` block stays below ~1 GiB whatever the model.  Differentiated by autograd."""
    x = qkv.view(B, S, n_head, 3, D)
    scale = 1.0 / math.sqrt(D)
    pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
    hidden = ~visible_mask(S, qkv.device, seg_start, B)
    group = max(1, min(n_head, (1 << 28) // max(1, B * S * S)))     # heads per block: <= 2^28 fp32 scores
    outs = []
    for h0 in range(0, n_head, group):
        h1 = min(n_head, h0 + group)
        q, k, v = (x[:, :, h0:h1, i].permute(0, 2, 1, 3) for i in range(3))      # [B, g, S, D] views
        scores = torch.matmul(q, k.transpose(-1, -2)).float() * scale
        scores = scores + slopes[h0:h1].float().view(1, -1, 1, 1) * pos.view(1, 1, 1, S)
        p = torch.softmax(scores.masked_fill(hidden, float("-inf")), dim=-1)
        p = torch.nn.functional.dropout(p, dropout_p, True).to(qkv.dtype)
        outs.append(torch.matmul(p, v))
    out = outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)
    return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D)


def native_seg_start(seg_start):
    """``seg_start`` as the flash kernels take it: contiguous int32 ``[B*S]`` (None stays None)."""
    return None if seg_start is None else seg_start.reshape(-1).to(torch.int32).contiguous()


class _AlibiAttentionNative(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, slopes, B, S, n_head, D, seg_start=None):
        out = torch.empty(B * S, n_head * D, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        seg = native_seg_start(seg_start)
        native().attention_fwd(qkv, slopes, out, lse, B, S, n_head, D, 0.0, seg)
        ctx.save_for_backward(qkv, slopes, out, lse, seg)
        ctx.dims = (B, S, n_head, D)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, slopes, out, lse, seg = ctx.saved_tensors
        B, S, n_head, D = ctx.dims
        dqkv = torch.empty_like(qkv)
        native().attention_bwd(qkv, slopes, out, lse, dout.contiguous(), dqkv, B, S, n_head, D, 0.0, seg)
        return dqkv, None, None, None, None, None, None


def _native_attention_available(D: int) -> bool:
    """Head sizes the flash kernel runs directly (no padding)."""
    return has_kernel("attention_fwd") and D in (64, 128)


def padded_head_dim(D: int) -> int:
    """The kernel's head width for a head of size ``D``: 64 or 128 (0: not supported)."""
    if D <= 64:
        return 64
    return 128 if D <= 128 else 0


def pad_heads(x: torch.Tensor, n_head: int, parts: int, D: int, DP: int) -> torch.Tensor:
    """``[tokens, n_head*parts*D] -> [tokens, n_head*parts*DP]``, every head (part) zero-padded from D to DP columns."""
    if D == DP:
        return x
    t = x.view(x.shape[0], n_head * parts, D)
    return torch.nn.functional.pad(t, (0, DP - D)).reshape(x.shape[0], n_head * parts * DP)


def unpad_heads(x: torch.Tensor, n_head: int, parts: int, D: int, DP: int) -> torch.Tensor:
    if D == DP:
        return x
    return x.view(x.shape[0], n_head * parts, DP)[..., :D].reshape(x.shape[0], n_head * parts * D)


class _AlibiAttentionPadded(torch.autograd.Function):
    """Head sizes the wgmma kernel has no tile shape for (e.g. D=80, bloom-3b): the heads are zero-padded to the
    next supported width and run through the same flash kernel with the softmax scale of the TRUE width — padded q/k
    columns add nothing to the scores, padded v columns produce output columns that are sliced away."""

    @staticmethod
    def forward(ctx, qkv, slopes, B, S, n_head, D, seg_start=None):
        DP = padded_head_dim(D)
        scale = 1.0 / math.sqrt(D)
        qkv_p = pad_heads(qkv, n_head, 3, D, DP).contiguous()
        out_p = torch.empty(B * S, n_head * DP, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        seg = native_seg_start(seg_start)
        native().attention_fwd(qkv_p, slopes, out_p, lse, B, S, n_head, DP, scale, seg)
        ctx.save_for_backward(qkv_p, slopes, out_p, lse, seg)
        ctx.dims = (B, S, n_head, D, DP, scale)
        return unpad_heads(out_p, n_head, 1, D, DP).contiguous()

    @staticmethod
    def backward(ctx, dout):
        qkv_p, slopes, out_p, lse, seg = ctx.saved_tensors
        B, S, n_head, D, DP, scale = ctx.dims
        dout_p = pad_heads(dout.contiguous(), n_head, 1, D, DP).contiguous()
        dqkv_p = torch.empty_like(qkv_p)
        native().attention_bwd(qkv_p, slopes, out_p, lse, dout_p, dqkv_p, B, S, n_head, DP, scale, seg)
        return unpad_heads(dqkv_p, n_head, 3, D, DP).contiguous(), None, None, None, None, None, None


def alibi_attention(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                    dropout_p: float = 0.0, seg_start=None) -> torch.Tensor:
    """``seg_start``: document starts of packed rows (module docstring), ``None``: one document per row."""
    if dropout_p > 0.0:
        return alibi_attention_with_dropout(qkv, slopes, B, S, n_head, D, dropout_p, seg_start=seg_start)
    if use_native(qkv) and _native_attention_available(D):
        return _AlibiAttentionNative.apply(qkv, slopes, B, S, n_head, D, seg_start)
    if use_native(qkv) and has_kernel("attention_fwd") and padded_head_dim(D) > 0 and D % 8 == 0:
        # e.g. D=80 (bloom-3b) on the D=128 kernel
        return _AlibiAttentionPadded.apply(qkv, slopes, B, S, n_head, D, seg_start)
    if qkv.is_cuda:
        # library fallback for head sizes beyond the kernel's widest tile (D > 128)
        x = qkv.view(B, S, n_head, 3, D)
        q, k, v = (x[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
        pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
        bias = slopes.float().view(1, n_head, 1, 1) * pos.view(1, 1, 1, S)
        visible = visible_mask(S, qkv.device, seg_start, B)
        rows = 1 if seg_start is None else B
        bias = bias.expand(rows, n_head, S, S).masked_fill(~visible, float("-inf")).to(qkv.dtype)
        out = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=bias)
        return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D)
    return alibi_attention_reference(qkv, slopes, B, S, n_head, D, seg_start=seg_start)


# ---------------------------------------------------------------------------------------------------------------------
# One decoding step against a preallocated KV cache.
#
# ``qkv_new`` is the step's QKV projection ``[B, n_head*3*D]`` (one token per row, same per-head layout as above),
# ``k_cache`` / ``v_cache`` are ``[B, n_head, capacity, D]``.  Every row appends its token at the same column ``pos``
# (a left-padded batch grows behind its last column).  The new k / v are written into ``cache[:, :, pos]``; row b's query
# then attends to keys ``lead[b] <= k <= pos`` with ``q.k * scale + slope[head] * (k - pos)``, which is the ALiBi
# score ``slope * k`` of the training path shifted by a per-row constant the softmax ignores.
# ---------------------------------------------------------------------------------------------------------------------

DECODE_HEAD_DIMS = (64, 80, 128)
_decode_tickets = {}


def alibi_decode_attention_reference(qkv_new: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
                                     slopes: torch.Tensor, pos: int, lead, D: int,
                                     softmax_scale: float = 0.0) -> torch.Tensor:
    """fp32 PyTorch form of :func:`alibi_decode_attention` (CPU path, test oracle).  ``lead``: int ``[B]`` leading pads
    per row or None; ``lead[b] > pos`` counts as ``pos``."""
    B, n_head, capacity = k_cache.shape[:3]
    if not 0 <= pos < capacity:
        raise ValueError(f"decode position {pos} is outside the cache capacity {capacity}")
    x = qkv_new.view(B, n_head, 3, D)
    k_cache[:, :, pos] = x[:, :, 1]
    v_cache[:, :, pos] = x[:, :, 2]
    q = x[:, :, 0].float()
    k, v = k_cache[:, :, :pos + 1].float(), v_cache[:, :, :pos + 1].float()
    scale = softmax_scale if softmax_scale > 0 else 1.0 / math.sqrt(D)
    scores = torch.einsum("bhd,bhkd->bhk", q, k) * scale
    key_pos = torch.arange(pos + 1, device=qkv_new.device)
    scores = scores + slopes.float().view(1, n_head, 1) * (key_pos - pos).float()
    if lead is not None:
        hidden = key_pos.view(1, 1, -1) < lead.to(key_pos.device).clamp(max=pos).view(-1, 1, 1)
        scores = scores.masked_fill(hidden, float("-inf"))
    out = torch.einsum("bhk,bhkd->bhd", scores.softmax(-1), v)
    return out.reshape(B, n_head * D).to(qkv_new.dtype)


def _decode_ticket(n: int, device) -> torch.Tensor:
    """The kernel's per-(row, head) arrival counters: zero between calls (the last CTA of each pair resets its own), so
    one zeroed array per device serves every call on that device's stream."""
    t = _decode_tickets.get(device)
    if t is None or t.numel() < n:
        t = torch.zeros(max(n, 4096), dtype=torch.int32, device=device)
        _decode_tickets[device] = t
    return t


def alibi_decode_attention(qkv_new: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, slopes: torch.Tensor,
                           pos: int, lead, D: int, softmax_scale: float = 0.0) -> torch.Tensor:
    """One decoding step (section comment above): returns ``[B, n_head*D]`` and writes the new keys and values into
    the caches.  CUDA bf16 inputs run the split-KV kernel (``csrc/decode_sm90.cu``, D in 64 / 80 / 128); ``lead`` is
    then an int tensor ``[B]`` on the same device, or None."""
    if not use_native(qkv_new):
        return alibi_decode_attention_reference(qkv_new, k_cache, v_cache, slopes, pos, lead, D, softmax_scale)
    if D not in DECODE_HEAD_DIMS:
        raise ValueError(f"the decode-attention kernel has no head size {D} (supported: {DECODE_HEAD_DIMS})")
    B, n_head, capacity = k_cache.shape[:3]
    if not 0 <= pos < capacity:
        raise ValueError(f"decode position {pos} is outside the cache capacity {capacity}")
    out = torch.empty(B, n_head * D, dtype=qkv_new.dtype, device=qkv_new.device)
    lead32 = None if lead is None else lead.to(torch.int32).contiguous()
    native().decode_attention(qkv_new.contiguous(), k_cache, v_cache, slopes.float().contiguous(), int(pos), lead32,
                              out, _decode_ticket(B * n_head, qkv_new.device), softmax_scale)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Paged KV cache (continuous batching, ``pipegoose_b200.serving``).
#
# ``k_pool`` / ``v_pool`` are ``[num_pages, n_head, PAGE_SIZE, D]``.  Row b's position p lives in page
# ``table[b, p // PAGE_SIZE]`` at slot ``p % PAGE_SIZE`` (``table``: int32 ``[B, max_pages]``).  Every row has its own
# new-token position ``pos[b]`` (int32 ``[B]``): the step writes its k / v into that slot, and row b's query attends to
# keys ``0 <= k <= pos[b]`` with ``q.k * scale + slope[head] * (k - pos[b])``.  ``max_pos`` is a host integer
# ``>= max(pos)``: it sizes the kernel's grid only.  Neither op reads ``table`` or ``pos`` on the host; their caller
# guarantees ``pos[b] <= max_pos`` and that the pages a row uses are pages of the pool.  The page holding ``pos[b]``
# belongs to row b alone; other pages may be shared between rows and are only read (prefix caching, beam search).
#
# FP8 pools (``ContinuousBatcher(kv_cache_dtype=torch.float8_e4m3fn)``): the pools hold ``torch.float8_e4m3fn`` codes
# and every op takes fp32 ``k_scales`` / ``v_scales`` ``[num_pages, n_head, PAGE_SIZE]``, one scale per position and
# head (:func:`quantize_kv` is the format).  Attention reads positions computed in earlier steps from the FP8 pools,
# dequantized, and positions computed in the same step from that step's ``qkv``, exactly: the decode op's key at
# ``pos[b]``, the prefill op's new tokens.
# ---------------------------------------------------------------------------------------------------------------------

PAGE_SIZE = 64
FP8_MAX = 448.0                         # largest finite float8_e4m3fn


def quantize_kv(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The FP8 pools' format: ``x [..., D]`` -> (``float8_e4m3fn`` codes ``[..., D]``, fp32 scales ``[...]``).  Per row,
    ``a = max |x|``, scale ``a / 448`` and codes ``e4m3_rn(x * (448 / a))`` (all 0 when ``a == 0``), in fp32 with IEEE
    division.  The kernels compute the same bits; no value exceeds 448 after the scaling, so nothing saturates."""
    x = x.float()
    a = x.abs().amax(-1, keepdim=True)
    m = torch.full_like(a, FP8_MAX)       # tensor / tensor: torch computes scalar / tensor as a reciprocal product
    codes = torch.where(a > 0, x * (m / a), torch.zeros_like(x)).to(torch.float8_e4m3fn)
    return codes, (a / m).squeeze(-1)


def dequantize_kv(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """fp32 values of FP8 pool rows: ``float(code) * scale``."""
    return codes.float() * scales.unsqueeze(-1)


def _fp8_pools(k_pool: torch.Tensor, k_scales, v_scales) -> bool:
    """Are these FP8 pools?  They need both scale tensors, and other pools take none."""
    fp8 = k_pool.dtype == torch.float8_e4m3fn
    if fp8 != (k_scales is not None) or (k_scales is None) != (v_scales is None):
        raise ValueError("float8_e4m3fn pools need k_scales and v_scales, and other pools take none")
    return fp8


def _paged_keys(pool: torch.Tensor, table: torch.Tensor, pos: torch.Tensor, n: int, scales=None):
    """fp32 ``pool`` rows of positions ``0 .. n-1`` of every table row as ``[B, n_head, n, D]`` (dequantized with
    ``scales`` from FP8 pools), zero behind ``pos[b]`` (a table row may hold anything behind its last used page, and
    unwritten slots anything at all), and the mask of the positions ``<= pos[b]``."""
    p = torch.arange(n, device=pool.device)
    valid = p.view(1, n) <= pos.view(-1, 1).to(p.dtype)
    pages = torch.where(valid, table.long()[:, p // PAGE_SIZE], torch.zeros_like(valid, dtype=torch.long))
    slots = (p % PAGE_SIZE).view(1, n)
    rows = pool[pages, :, slots].float() if scales is None else dequantize_kv(pool[pages, :, slots],
                                                                              scales[pages, :, slots])
    rows = rows.masked_fill(~valid.view(*valid.shape, 1, 1), 0.0)
    return rows.transpose(1, 2), valid


def _store_kv(k: torch.Tensor, v: torch.Tensor, page: torch.Tensor, off: torch.Tensor, k_pool: torch.Tensor,
              v_pool: torch.Tensor, k_scales, v_scales) -> None:
    """``k`` / ``v [n, n_head, D]`` into slot ``off[i]`` of page ``page[i]``, quantized into FP8 pools."""
    if k_scales is None:
        k_pool[page, :, off] = k.to(k_pool.dtype)
        v_pool[page, :, off] = v.to(v_pool.dtype)
        return
    for x, pool, scales in ((k, k_pool, k_scales), (v, v_pool, v_scales)):
        codes, s = quantize_kv(x)
        pool[page, :, off] = codes.to(pool.device)
        scales[page, :, off] = s.to(scales.device)


def _check_max_pos(max_pos: int, table: torch.Tensor) -> None:
    if not 0 <= max_pos < table.shape[1] * PAGE_SIZE:
        raise ValueError(f"max_pos {max_pos} is outside the {table.shape[1]} pages of a table row")


def alibi_paged_decode_attention_reference(qkv_new: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                                           table: torch.Tensor, pos: torch.Tensor, max_pos: int, slopes: torch.Tensor,
                                           D: int, softmax_scale: float = 0.0, k_scales=None,
                                           v_scales=None) -> torch.Tensor:
    """fp32 PyTorch form of :func:`alibi_paged_decode_attention` (CPU path, test oracle)."""
    fp8 = _fp8_pools(k_pool, k_scales, v_scales)
    _check_max_pos(max_pos, table)
    B, n_head = table.shape[0], k_pool.shape[1]
    if B == 0:
        return qkv_new.new_empty(0, n_head * D)
    x = qkv_new.view(B, n_head, 3, D)
    pos = pos.to(table.device).long()
    page = table.long().gather(1, (pos // PAGE_SIZE).view(B, 1)).view(B)
    _store_kv(x[:, :, 1], x[:, :, 2], page, pos % PAGE_SIZE, k_pool, v_pool, k_scales, v_scales)
    k, valid = _paged_keys(k_pool, table, pos, max_pos + 1, k_scales)
    v, _ = _paged_keys(v_pool, table, pos, max_pos + 1, v_scales)
    if fp8:                                                     # the step's own key and value: exact
        rows = torch.arange(B, device=k.device)
        k[rows, :, pos.to(k.device)] = x[:, :, 1].float().to(k.device)
        v[rows, :, pos.to(k.device)] = x[:, :, 2].float().to(k.device)
    scale = softmax_scale if softmax_scale > 0 else 1.0 / math.sqrt(D)
    scores = torch.einsum("bhd,bhkd->bhk", x[:, :, 0].float(), k) * scale
    key_pos = torch.arange(max_pos + 1, device=k_pool.device)
    scores = scores + slopes.float().view(1, n_head, 1) * (key_pos.view(1, 1, -1) - pos.view(B, 1, 1)).float()
    scores = scores.masked_fill(~valid.view(B, 1, -1), float("-inf"))
    out = torch.einsum("bhk,bhkd->bhd", scores.softmax(-1), v)
    return out.reshape(B, n_head * D).to(qkv_new.dtype)


def alibi_paged_decode_attention(qkv_new: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                                 table: torch.Tensor, pos: torch.Tensor, max_pos: int, slopes: torch.Tensor, D: int,
                                 softmax_scale: float = 0.0, k_scales=None, v_scales=None, out=None) -> torch.Tensor:
    """One decoding step of ``B`` independent sequences over the paged pools (section comment above): returns
    ``[B, n_head*D]`` and writes the new keys and values into the pools.  CUDA bf16 inputs run the paged form of the
    split-KV kernel (``csrc/decode_sm90.cu``, D in 64 / 80 / 128), or its FP8 form over FP8 pools; ``out`` (contiguous
    ``[B, n_head*D]``, kernel path only) receives the result instead of a new tensor."""
    fp8 = _fp8_pools(k_pool, k_scales, v_scales)
    if not use_native(qkv_new):
        return alibi_paged_decode_attention_reference(qkv_new, k_pool, v_pool, table, pos, max_pos, slopes, D,
                                                      softmax_scale, k_scales=k_scales, v_scales=v_scales)
    if D not in DECODE_HEAD_DIMS:
        raise ValueError(f"the decode-attention kernel has no head size {D} (supported: {DECODE_HEAD_DIMS})")
    _check_max_pos(max_pos, table)
    B, n_head = table.shape[0], k_pool.shape[1]
    if out is None:
        out = torch.empty(B, n_head * D, dtype=qkv_new.dtype, device=qkv_new.device)
    table, pos = table.to(torch.int32).contiguous(), pos.to(torch.int32).contiguous()
    ticket = _decode_ticket(B * n_head, qkv_new.device)
    if fp8:
        native().paged_decode_attention_fp8(qkv_new.contiguous(), k_pool, v_pool, k_scales, v_scales, table, pos,
                                            int(max_pos), slopes.float().contiguous(), out, ticket, softmax_scale)
    else:
        native().paged_decode_attention(qkv_new.contiguous(), k_pool, v_pool, table, pos, int(max_pos),
                                        slopes.float().contiguous(), out, ticket, softmax_scale)
    return out


def paged_kv_write_reference(qkv: torch.Tensor, slot: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                             D: int, k_scales=None, v_scales=None) -> None:
    """PyTorch form of :func:`paged_kv_write`."""
    _fp8_pools(k_pool, k_scales, v_scales)
    n_head = k_pool.shape[1]
    x = qkv.view(-1, n_head, 3, D)
    slot = slot.to(k_pool.device).long()
    _store_kv(x[:, :, 1], x[:, :, 2], slot // PAGE_SIZE, slot % PAGE_SIZE, k_pool, v_pool, k_scales, v_scales)


def paged_kv_write(qkv: torch.Tensor, slot: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, D: int,
                   k_scales=None, v_scales=None) -> None:
    """Prefill: the keys and values of every token ``n`` of ``qkv [N, n_head*3*D]`` into pool slot ``slot[n]``
    (``page * PAGE_SIZE + offset``, int32 ``[N]``) for every head, quantized into FP8 pools.  CUDA bf16 inputs run
    ``paged_kv_write_kernel`` (``paged_kv_write_fp8_kernel``)."""
    fp8 = _fp8_pools(k_pool, k_scales, v_scales)
    if not use_native(qkv):
        return paged_kv_write_reference(qkv, slot, k_pool, v_pool, D, k_scales, v_scales)
    if D not in DECODE_HEAD_DIMS:
        raise ValueError(f"the paged KV cache has no head size {D} (supported: {DECODE_HEAD_DIMS})")
    if fp8:
        native().paged_kv_write_fp8(qkv.contiguous(), slot.to(torch.int32).contiguous(), k_pool, v_pool, k_scales,
                                    v_scales)
    else:
        native().paged_kv_write(qkv.contiguous(), slot.to(torch.int32).contiguous(), k_pool, v_pool)


def paged_kv_dequantize_reference(k_pool: torch.Tensor, v_pool: torch.Tensor, k_scales: torch.Tensor,
                                  v_scales: torch.Tensor, src: torch.Tensor, dst: torch.Tensor, k_out: torch.Tensor,
                                  v_out: torch.Tensor) -> None:
    """PyTorch form of :func:`paged_kv_dequantize`."""
    src, dst = src.long().to(k_pool.device), dst.long().to(k_out.device)
    k_out[dst] = dequantize_kv(k_pool[src], k_scales[src]).to(k_out.dtype).to(k_out.device)
    v_out[dst] = dequantize_kv(v_pool[src], v_scales[src]).to(v_out.dtype).to(v_out.device)


def paged_kv_dequantize(k_pool: torch.Tensor, v_pool: torch.Tensor, k_scales: torch.Tensor, v_scales: torch.Tensor,
                        src: torch.Tensor, dst: torch.Tensor, k_out: torch.Tensor, v_out: torch.Tensor) -> None:
    """Pages ``src[i]`` of FP8 pools, dequantized, into pages ``dst[i]`` of ``k_out`` / ``v_out [*, n_head,
    PAGE_SIZE, D]`` (int32 page lists).  CUDA bf16 outputs run ``kv_dequantize_kernel``."""
    if not use_native(k_out):
        return paged_kv_dequantize_reference(k_pool, v_pool, k_scales, v_scales, src, dst, k_out, v_out)
    native().paged_kv_dequantize(k_pool, v_pool, k_scales, v_scales, src.to(torch.int32).contiguous(),
                                 dst.to(torch.int32).contiguous(), k_out, v_out)


def _copy_pairs(pairs) -> torch.Tensor:
    return (pairs if torch.is_tensor(pairs) else torch.tensor(pairs, dtype=torch.int32)).to(torch.int32).view(-1, 3)


def paged_kv_copy_reference(pairs, k_pools: torch.Tensor, v_pools: torch.Tensor, k_scales=None,
                            v_scales=None) -> None:
    """PyTorch form of :func:`paged_kv_copy`."""
    _fp8_pools(k_pools, k_scales, v_scales)
    for src, dst, n in _copy_pairs(pairs).tolist():
        for t in (k_pools, v_pools) + ((k_scales, v_scales) if k_scales is not None else ()):
            t[:, dst, :, :n] = t[:, src, :, :n]


def paged_kv_copy(pairs, k_pools: torch.Tensor, v_pools: torch.Tensor, k_scales=None, v_scales=None) -> None:
    """Beam-search forks: for every ``(src page, dst page, count)`` of ``pairs`` (int32 ``[n, 3]`` or a host list of
    triples) and every layer of the pools ``[n_layer, pages, n_head, PAGE_SIZE, D]``, slots ``0 .. count-1`` of page
    ``src`` into page ``dst``, with their scales ``[n_layer, pages, n_head, PAGE_SIZE]`` over FP8 pools; nothing else
    changes.  No ``dst`` may also be a ``src``.  CUDA bf16 and FP8 pools run ``paged_kv_copy_kernel``, one launch for
    all pairs and layers."""
    fp8 = _fp8_pools(k_pools, k_scales, v_scales)
    if not (k_pools.is_cuda and (fp8 or k_pools.dtype == torch.bfloat16)):
        return paged_kv_copy_reference(pairs, k_pools, v_pools, k_scales, v_scales)
    pairs = _copy_pairs(pairs).to(k_pools.device, non_blocking=True).contiguous()
    native().paged_kv_copy(pairs, k_pools, v_pools, k_scales, v_scales)


def _swap_pairs(pairs, pages: int, slots: int) -> torch.Tensor:
    """``pairs`` as int32 ``[n, 2]``; a host list or CPU tensor is checked against the pool and host-pool sizes (a CUDA
    tensor is the caller's to get right: checking it would synchronise)."""
    pairs = (pairs if torch.is_tensor(pairs) else torch.tensor(pairs, dtype=torch.int32)).to(torch.int32).view(-1, 2)
    if not pairs.is_cuda and pairs.numel() and not (0 <= int(pairs[:, 0].min()) and int(pairs[:, 0].max()) < pages and
                                                    0 <= int(pairs[:, 1].min()) and int(pairs[:, 1].max()) < slots):
        raise ValueError(f"paged_kv_swap: pairs {pairs.tolist()} outside the pool's {pages} pages or the host pool's "
                         f"{slots} slots")
    return pairs


def paged_kv_swap_reference(pairs, k_pools: torch.Tensor, v_pools: torch.Tensor, k_scales, v_scales,
                            host_kv: torch.Tensor, host_scales, to_host: bool) -> None:
    """PyTorch form of :func:`paged_kv_swap` (bytes copied as they are, so FP8 codes move bit for bit)."""
    fp8 = _fp8_pools(k_pools, k_scales, v_scales)
    if fp8 != (host_scales is not None):
        raise ValueError("float8_e4m3fn pools need host_scales, and other pools take none")
    pools = [(k_pools, host_kv[:, :, 0]), (v_pools, host_kv[:, :, 1])]
    if fp8:
        pools += [(k_scales, host_scales[:, :, 0]), (v_scales, host_scales[:, :, 1])]
    for page, slot in _swap_pairs(pairs, k_pools.shape[1], host_kv.shape[0]).tolist():
        for pool, host in pools:
            if to_host:
                host[slot].copy_(pool[:, page])
            else:
                pool[:, page].copy_(host[slot])


def paged_kv_swap(pairs, k_pools: torch.Tensor, v_pools: torch.Tensor, k_scales, v_scales, host_kv: torch.Tensor,
                  host_scales, to_host: bool) -> None:
    """Preemption: for every ``(pool page, host slot)`` of ``pairs`` (int32 ``[n, 2]`` or a host list of pairs), every
    layer's K and V of page ``page`` of the pools ``[n_layer, pages, n_head, PAGE_SIZE, D]`` to (``to_host``) or from
    slot ``slot`` of ``host_kv [slots, n_layer, 2, n_head, PAGE_SIZE, D]``, and over FP8 pools the scales ``[n_layer,
    pages, n_head, PAGE_SIZE]`` to or from ``host_scales [slots, n_layer, 2, n_head, PAGE_SIZE]`` (fp32; ``None`` for
    other pools); nothing else changes.  No page or slot may appear twice.  CUDA bf16 and FP8 pools run
    ``paged_kv_swap_kernel``, one launch for all pairs and layers, which reads and writes the host pool (pinned: refused
    otherwise) through its device pointer, in stream order; the host must not touch the host pool meanwhile."""
    fp8 = _fp8_pools(k_pools, k_scales, v_scales)
    if not (k_pools.is_cuda and (fp8 or k_pools.dtype == torch.bfloat16)):
        return paged_kv_swap_reference(pairs, k_pools, v_pools, k_scales, v_scales, host_kv, host_scales, to_host)
    pairs = _swap_pairs(pairs, k_pools.shape[1], host_kv.shape[0]).to(k_pools.device, non_blocking=True).contiguous()
    native().paged_kv_swap(pairs, k_pools, v_pools, k_scales, v_scales, host_kv, host_scales, bool(to_host))


# ---------------------------------------------------------------------------------------------------------------------
# Prefill against paged pools (prefix caching, ``pipegoose_b200.serving``).
#
# ``qkv [N, n_head*3*D]`` holds the new tokens of R sequences packed back to back: sequence r owns rows
# ``cu_seqlens[r] .. cu_seqlens[r+1]-1`` (int32 ``[R+1]``), and its first new token sits at position ``start[r]`` (int32
# ``[R]``), so row n is at ``p = start[r] + n - cu_seqlens[r]``.  Its query attends to keys ``0 <= k <= p`` of sequence r,
# all read from the pools through ``table`` (int32 ``[R, max_pages]``) with ``q.k * scale + slope[head] * (k - p)``: the
# cached prefix and the new tokens are read the same way, so the caller stores the new keys and values with
# :func:`paged_kv_write` first.  The op does not write the pools.  ``max_len`` is a host integer ``>= `` every sequence's
# new tokens: it sizes the kernel's grid only.  The kernel does not read ``cu_seqlens`` / ``start`` on the host and
# trusts them (as the decode op trusts ``pos``); it checks ``max_len`` against them only when they are host tensors.
#
# FP8 pools: the new tokens are read from ``qkv`` (the rule of the section above), the cached prefix from the pools.
# Every ``start[r]`` is then a multiple of PAGE_SIZE (prefix caching shares full pages only, chunked prefill cuts
# prompts at page boundaries), so the kernel runs on a step-local bf16 staging pool that holds just the step's
# sequences (:func:`fp8_prefill_staging`): their cached pages dequantized, then their new tokens' exact keys and values.
# ---------------------------------------------------------------------------------------------------------------------

def _check_prefill_bounds(cu_seqlens: torch.Tensor, max_len: int, table: torch.Tensor, D: int = 0) -> None:
    if D and D not in DECODE_HEAD_DIMS:
        raise ValueError(f"the paged prefill-attention kernel has no head size {D} (supported: {DECODE_HEAD_DIMS})")
    if not 1 <= max_len <= table.shape[1] * PAGE_SIZE:
        raise ValueError(f"max_len {max_len} is outside 1 .. the {table.shape[1] * PAGE_SIZE} positions of a table row")
    if not cu_seqlens.is_cuda and cu_seqlens.numel() > 1:         # host data: checked without a device sync
        longest = int((cu_seqlens[1:] - cu_seqlens[:-1]).max())
        if longest > max_len:
            raise ValueError(f"max_len {max_len} is smaller than the longest sequence ({longest} new tokens)")


def alibi_paged_prefill_attention_reference(qkv: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                                            table: torch.Tensor, cu_seqlens: torch.Tensor, start: torch.Tensor,
                                            max_len: int, slopes: torch.Tensor, D: int,
                                            softmax_scale: float = 0.0, k_scales=None, v_scales=None) -> torch.Tensor:
    """fp32 PyTorch form of :func:`alibi_paged_prefill_attention` (CPU path, test oracle).  Reads ``cu_seqlens`` and
    ``start`` on the host.  No pool slot past a sequence's last position reaches the result."""
    _check_prefill_bounds(cu_seqlens.cpu(), max_len, table, D)
    return paged_prefill_attention_fp32(qkv, k_pool, v_pool, table, cu_seqlens, start, max_len, slopes, D,
                                        softmax_scale, k_scales=k_scales, v_scales=v_scales)


def paged_prefill_attention_fp32(qkv: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, table: torch.Tensor,
                                 cu_seqlens: torch.Tensor, start: torch.Tensor, max_len: int, slopes: torch.Tensor,
                                 D: int, softmax_scale: float = 0.0, k_scales=None, v_scales=None) -> torch.Tensor:
    """The reference's computation for any head size (the model's path where no kernel has its head size)."""
    fp8 = _fp8_pools(k_pool, k_scales, v_scales)
    _check_prefill_bounds(cu_seqlens.cpu(), max_len, table)
    n_head = k_pool.shape[1]
    N = qkv.shape[0]
    out = torch.zeros(N, n_head, D, dtype=torch.float32, device=qkv.device)
    cu, st = cu_seqlens.tolist(), start.tolist()
    scale = softmax_scale if softmax_scale > 0 else 1.0 / math.sqrt(D)
    for r in range(len(st)):
        n0, n1 = cu[r], cu[r + 1]
        if n1 == n0:
            continue
        last = st[r] + n1 - n0 - 1                                   # the sequence's last position
        pos = torch.tensor([last], device=k_pool.device)
        k, _ = _paged_keys(k_pool, table[r:r + 1], pos, last + 1, k_scales)   # [1, H, last+1, D], zero past `last`
        v, _ = _paged_keys(v_pool, table[r:r + 1], pos, last + 1, v_scales)
        x = qkv[n0:n1].view(n1 - n0, n_head, 3, D).float().transpose(0, 1).to(k.device)         # [H, n, 3, D]
        if fp8:                                                      # the new tokens: exact
            k[0, :, st[r]:] = x[:, :, 1]
            v[0, :, st[r]:] = x[:, :, 2]
        q = x[:, :, 0]
        scores = torch.matmul(q, k[0].transpose(-1, -2)) * scale    # [H, n, last+1]
        qp = torch.arange(st[r], last + 1, device=k.device).view(1, -1, 1)
        kp = torch.arange(last + 1, device=k.device).view(1, 1, -1)
        scores = scores + slopes.float().to(k.device).view(n_head, 1, 1) * (kp - qp).float()
        scores = scores.masked_fill(kp > qp, float("-inf"))
        out[n0:n1] = torch.matmul(scores.softmax(-1), v[0]).transpose(0, 1).to(out.device)
    return out.reshape(N, n_head * D).to(qkv.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# Append to paged pools (speculative verification, ``pipegoose_b200.serving``).
#
# Row r of ``table`` appends ``n_r = cu_seqlens[r+1] - cu_seqlens[r]`` tokens, ``1 <= n_r <= APPEND_MAX_TOKENS``,
# packed in ``qkv [N, n_head*3*D]`` at positions ``pos[r] .. pos[r] + n_r - 1``.  The op writes their keys and values
# into their slots, and query i of row r attends to keys ``0 .. pos[r] + i`` with ``q.k * scale + slope[head] *
# (k - (pos[r] + i))``.  ``max_pos`` is a host integer ``>= pos[r] + n_r - 1`` for every row: it sizes the grid only.
# ``max_tokens`` is a host integer ``>= n_r`` for every row: it picks the kernel's query tile.  Like the decode op, the
# kernel reads ``table``, ``cu_seqlens`` and ``pos`` on the device only and trusts them; the row lengths, ``max_pos``
# and ``max_tokens`` are checked against them when they are host tensors.  Its reference is the prefill reference after
# the pool write.  FP8 pools are not supported.
# ---------------------------------------------------------------------------------------------------------------------

APPEND_MAX_TOKENS = 8


def _append_tile(cu_seqlens: torch.Tensor, pos: torch.Tensor, max_pos: int, max_tokens: int, N: int, B: int) -> int:
    """Checks what the host can see and returns the bound on the rows' token counts: ``max_tokens``, or when it is 0
    the longest row of host ``cu_seqlens`` (of device ones: ``N - B + 1``, every row appending at least one token)."""
    if not 0 <= max_tokens <= APPEND_MAX_TOKENS:
        raise ValueError(f"max_tokens {max_tokens} is outside 1 .. {APPEND_MAX_TOKENS} (0: from cu_seqlens)")
    if cu_seqlens.is_cuda or pos.is_cuda or B == 0:
        return max_tokens or max(1, min(APPEND_MAX_TOKENS, N - B + 1))
    n = cu_seqlens[1:] - cu_seqlens[:-1]
    if not bool(((n >= 1) & (n <= APPEND_MAX_TOKENS)).all()):
        raise ValueError(f"every row appends 1 .. {APPEND_MAX_TOKENS} tokens, got {n.tolist()}")
    longest = int(n.max())
    if max_tokens and longest > max_tokens:
        raise ValueError(f"max_tokens {max_tokens} is smaller than the longest row ({longest} tokens)")
    last = int((pos.long() + n.long()).max()) - 1
    if last > max_pos:
        raise ValueError(f"max_pos {max_pos} is smaller than the last appended position {last}")
    return max_tokens or longest


def alibi_paged_append_attention_reference(qkv: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                                           table: torch.Tensor, cu_seqlens: torch.Tensor, pos: torch.Tensor,
                                           max_pos: int, slopes: torch.Tensor, D: int, softmax_scale: float = 0.0,
                                           max_tokens: int = 0) -> torch.Tensor:
    """PyTorch form of :func:`alibi_paged_append_attention` for any head size (CPU path, test oracle, and the model's
    path where no kernel has its head size): :func:`paged_kv_write_reference` of the new tokens, then
    :func:`paged_prefill_attention_fp32` from ``start = pos``.  Reads ``cu_seqlens`` and ``pos`` on the host."""
    if k_pool.dtype == torch.float8_e4m3fn:
        raise ValueError("append attention does not support FP8 pools")
    _check_max_pos(max_pos, table)
    B = table.shape[0]
    cu_seqlens, pos = cu_seqlens.cpu(), pos.cpu()
    longest = _append_tile(cu_seqlens, pos, max_pos, max_tokens, qkv.shape[0], B)
    cu, st = cu_seqlens.tolist(), pos.tolist()
    rows = table.cpu().tolist()
    slot = [rows[r][p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE
            for r in range(B) for p in range(st[r], st[r] + cu[r + 1] - cu[r])]
    paged_kv_write_reference(qkv, torch.tensor(slot, dtype=torch.long), k_pool, v_pool, D)
    return paged_prefill_attention_fp32(qkv, k_pool, v_pool, table, cu_seqlens, pos, longest, slopes, D,
                                        softmax_scale)


def alibi_paged_append_attention(qkv: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, table: torch.Tensor,
                                 cu_seqlens: torch.Tensor, pos: torch.Tensor, max_pos: int, slopes: torch.Tensor,
                                 D: int, softmax_scale: float = 0.0, max_tokens: int = 0) -> torch.Tensor:
    """Append the tokens of every row to the paged pools and attend (section comment above): returns
    ``[N, n_head*D]``.  CUDA bf16 inputs run ``append_attention_kernel`` (``csrc/decode_sm90.cu``, D in 64 / 80 / 128);
    otherwise :func:`alibi_paged_append_attention_reference` runs.  ``max_tokens`` (1 .. 8) is a host bound on every
    row's token count that picks the kernel's query tile (1, 2, 4 or 8 queries per CTA, each costing registers for
    every row); 0 takes the longest row of host ``cu_seqlens``, or ``N - B + 1`` for device ones."""
    if not use_native(qkv):
        return alibi_paged_append_attention_reference(qkv, k_pool, v_pool, table, cu_seqlens, pos, max_pos, slopes, D,
                                                      softmax_scale, max_tokens)
    if k_pool.dtype == torch.float8_e4m3fn:
        raise ValueError("append attention does not support FP8 pools")
    if D not in DECODE_HEAD_DIMS:
        raise ValueError(f"the append-attention kernel has no head size {D} (supported: {DECODE_HEAD_DIMS})")
    _check_max_pos(max_pos, table)
    B, n_head = table.shape[0], k_pool.shape[1]
    tile = _append_tile(cu_seqlens, pos, max_pos, max_tokens, qkv.shape[0], B)
    out = torch.empty(qkv.shape[0], n_head * D, dtype=qkv.dtype, device=qkv.device)
    native().paged_append_attention(qkv.contiguous(), k_pool, v_pool, table.to(torch.int32).contiguous(),
                                    cu_seqlens.to(qkv.device, torch.int32).contiguous(),
                                    pos.to(qkv.device, torch.int32).contiguous(), int(max_pos), tile,
                                    slopes.float().contiguous(), out,
                                    _decode_ticket(APPEND_MAX_TOKENS * B * n_head, qkv.device), softmax_scale)
    return out


def fp8_prefill_staging(pages, cached, lengths):
    """Host plan of a prefill with cached prefixes over FP8 pools.  Sequence r has pool pages ``pages[r]``, its first
    ``cached[r]`` positions (a multiple of PAGE_SIZE) in the pools and ``lengths[r]`` positions in all; it gets staging
    pages ``o_r .. o_r + ceil(lengths[r] / PAGE_SIZE) - 1``.  Returns ``(num_pages, src, dst, slot, table)``: the
    staging pool's size, its cached pages' pool ids ``src`` and staging ids ``dst``, the staging slot of every new
    token (in sequence order) and the staging table rows (int lists, padded with page 0)."""
    src, dst, slot, rows, o = [], [], [], [], 0
    for pg, c, n in zip(pages, cached, lengths):
        if c % PAGE_SIZE:
            raise ValueError(f"a cached prefix of {c} positions is not a whole number of pages")
        need = -(-n // PAGE_SIZE)
        src += pg[:c // PAGE_SIZE]
        dst += range(o, o + c // PAGE_SIZE)
        slot += range(o * PAGE_SIZE + c, o * PAGE_SIZE + n)
        rows.append(list(range(o, o + need)))
        o += need
    width = max((len(r) for r in rows), default=1)
    return o, src, dst, slot, [r + [0] * (width - len(r)) for r in rows]


def alibi_paged_prefill_attention(qkv: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, table: torch.Tensor,
                                  cu_seqlens: torch.Tensor, start: torch.Tensor, max_len: int, slopes: torch.Tensor,
                                  D: int, softmax_scale: float = 0.0, k_scales=None, v_scales=None,
                                  stage=None, out=None) -> torch.Tensor:
    """Attention of the new tokens of R sequences over their paged keys (section comment above): returns
    ``[N, n_head*D]``.  CUDA bf16 inputs run the paged form of the flash kernel (``csrc/attention_sm90.cu``, D in
    64 / 80 / 128; D = 80 on the D = 128 instantiation without padded copies).

    Over FP8 pools the kernel reads a bf16 staging pool: ``stage = (k_stage, v_stage, src, dst, slot, table)``, the
    staging pools ``[>= num_pages, n_head, PAGE_SIZE, D]`` (their content is overwritten) and the device int32 lists
    of :func:`fp8_prefill_staging` (``table`` as ``[R, width]``).  The reference path needs no ``stage``.  ``out``
    (contiguous ``[N, n_head*D]``, kernel path only) receives the result instead of a new tensor."""
    fp8 = _fp8_pools(k_pool, k_scales, v_scales)
    if not use_native(qkv):
        return alibi_paged_prefill_attention_reference(qkv, k_pool, v_pool, table, cu_seqlens, start, max_len, slopes,
                                                       D, softmax_scale, k_scales=k_scales, v_scales=v_scales)
    if fp8:
        if stage is None:
            raise ValueError("the paged prefill kernel reads FP8 pools through a staging pool: pass stage")
        k_stage, v_stage, src, dst, slot, table = stage
        paged_kv_dequantize(k_pool, v_pool, k_scales, v_scales, src, dst, k_stage, v_stage)
        paged_kv_write(qkv, slot, k_stage, v_stage, D)
        k_pool, v_pool = k_stage, v_stage
    _check_prefill_bounds(cu_seqlens, max_len, table, D)
    n_head = k_pool.shape[1]
    if out is None:
        out = torch.empty(qkv.shape[0], n_head * D, dtype=qkv.dtype, device=qkv.device)
    native().paged_prefill_attention(qkv.contiguous(), k_pool, v_pool, table.to(torch.int32).contiguous(),
                                     cu_seqlens.to(qkv.device, torch.int32).contiguous(),
                                     start.to(qkv.device, torch.int32).contiguous(), int(max_len),
                                     slopes.float().contiguous(), out, softmax_scale)
    return out
