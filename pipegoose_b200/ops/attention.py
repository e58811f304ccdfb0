"""Causal ALiBi self-attention on Bloom's fused QKV layout.

``qkv`` is ``[B*S, n_head*3*D]`` with each row laid out ``[head][q|k|v][D]`` (the layout HF Bloom's
``query_key_value`` produces), the result is ``[B*S, n_head*D]``.  Scores are
``q.k / sqrt(D) + slope[head] * key_position`` under a causal mask, softmax in fp32.

Two implementations share this contract: the sm_90a flash kernel (``csrc/attention_sm90.cu``:
wgmma QK^T / PV with register accumulators, online softmax, never materialising ``[S, S]``) and
the PyTorch reference below (CPU tests, numerics oracle).
"""
from __future__ import annotations

import math

import torch

from pipegoose_b200.ops import has_kernel, native, use_native


def alibi_attention_reference(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                              softmax_scale: float = 0.0, dropout_p: float = 0.0) -> torch.Tensor:
    """``dropout_p > 0``: dropout on the attention probabilities (🤗 Bloom's ``attention_dropout``: zeroed entries, the
    rest scaled by ``1 / (1 - p)``, rows not re-normalised)."""
    x = qkv.view(B, S, n_head, 3, D)
    q, k, v = (x[:, :, :, i].permute(0, 2, 1, 3).float() for i in range(3))  # [B, H, S, D]
    scores = torch.matmul(q, k.transpose(-1, -2)) * (softmax_scale if softmax_scale > 0 else 1.0 / math.sqrt(D))
    pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
    scores = scores + slopes.float().view(1, n_head, 1, 1) * pos.view(1, 1, 1, S)
    causal = torch.ones(S, S, dtype=torch.bool, device=qkv.device).tril()
    scores = scores.masked_fill(~causal, float("-inf"))
    p = torch.softmax(scores, dim=-1)
    if dropout_p > 0.0:
        p = torch.nn.functional.dropout(p, dropout_p, True)
    out = torch.matmul(p, v)  # [B, H, S, D]
    return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D).to(qkv.dtype)


def alibi_attention_with_dropout(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                                 dropout_p: float) -> torch.Tensor:
    """Training-time attention with dropout on the probabilities.  The flash kernel never holds a row of probabilities
    (online softmax), so this path materialises them: bf16 GEMMs around an fp32 softmax, one head group at a time so
    that the live ``[B, heads, S, S]`` block stays below ~1 GiB whatever the model.  Differentiated by autograd."""
    x = qkv.view(B, S, n_head, 3, D)
    scale = 1.0 / math.sqrt(D)
    pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
    causal = torch.ones(S, S, dtype=torch.bool, device=qkv.device).tril()
    group = max(1, min(n_head, (1 << 28) // max(1, B * S * S)))     # heads per block: <= 2^28 fp32 scores
    outs = []
    for h0 in range(0, n_head, group):
        h1 = min(n_head, h0 + group)
        q, k, v = (x[:, :, h0:h1, i].permute(0, 2, 1, 3) for i in range(3))      # [B, g, S, D] views
        scores = torch.matmul(q, k.transpose(-1, -2)).float() * scale
        scores = scores + slopes[h0:h1].float().view(1, -1, 1, 1) * pos.view(1, 1, 1, S)
        p = torch.softmax(scores.masked_fill(~causal, float("-inf")), dim=-1)
        p = torch.nn.functional.dropout(p, dropout_p, True).to(qkv.dtype)
        outs.append(torch.matmul(p, v))
    out = outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)
    return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D)


class _AlibiAttentionNative(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, slopes, B, S, n_head, D):
        out = torch.empty(B * S, n_head * D, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        native().attention_fwd(qkv, slopes, out, lse, B, S, n_head, D)
        ctx.save_for_backward(qkv, slopes, out, lse)
        ctx.dims = (B, S, n_head, D)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, slopes, out, lse = ctx.saved_tensors
        B, S, n_head, D = ctx.dims
        dqkv = torch.empty_like(qkv)
        native().attention_bwd(qkv, slopes, out, lse, dout.contiguous(), dqkv, B, S, n_head, D)
        return dqkv, None, None, None, None, None


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
    def forward(ctx, qkv, slopes, B, S, n_head, D):
        DP = padded_head_dim(D)
        scale = 1.0 / math.sqrt(D)
        qkv_p = pad_heads(qkv, n_head, 3, D, DP).contiguous()
        out_p = torch.empty(B * S, n_head * DP, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        native().attention_fwd(qkv_p, slopes, out_p, lse, B, S, n_head, DP, scale)
        ctx.save_for_backward(qkv_p, slopes, out_p, lse)
        ctx.dims = (B, S, n_head, D, DP, scale)
        return unpad_heads(out_p, n_head, 1, D, DP).contiguous()

    @staticmethod
    def backward(ctx, dout):
        qkv_p, slopes, out_p, lse = ctx.saved_tensors
        B, S, n_head, D, DP, scale = ctx.dims
        dout_p = pad_heads(dout.contiguous(), n_head, 1, D, DP).contiguous()
        dqkv_p = torch.empty_like(qkv_p)
        native().attention_bwd(qkv_p, slopes, out_p, lse, dout_p, dqkv_p, B, S, n_head, DP, scale)
        return unpad_heads(dqkv_p, n_head, 3, D, DP).contiguous(), None, None, None, None, None


def alibi_attention(qkv: torch.Tensor, slopes: torch.Tensor, B: int, S: int, n_head: int, D: int,
                    dropout_p: float = 0.0) -> torch.Tensor:
    if dropout_p > 0.0:
        return alibi_attention_with_dropout(qkv, slopes, B, S, n_head, D, dropout_p)
    if use_native(qkv) and _native_attention_available(D):
        return _AlibiAttentionNative.apply(qkv, slopes, B, S, n_head, D)
    if use_native(qkv) and has_kernel("attention_fwd") and padded_head_dim(D) > 0 and D % 8 == 0:
        return _AlibiAttentionPadded.apply(qkv, slopes, B, S, n_head, D)  # e.g. D=80 (bloom-3b) on the D=128 kernel
    if qkv.is_cuda:
        # library fallback for head sizes beyond the kernel's widest tile (D > 128)
        x = qkv.view(B, S, n_head, 3, D)
        q, k, v = (x[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
        pos = torch.arange(S, device=qkv.device, dtype=torch.float32)
        bias = slopes.float().view(1, n_head, 1, 1) * pos.view(1, 1, 1, S)
        causal = torch.ones(S, S, dtype=torch.bool, device=qkv.device).tril()
        bias = bias.expand(1, n_head, S, S).masked_fill(~causal, float("-inf")).to(qkv.dtype)
        out = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=bias)
        return out.permute(0, 2, 1, 3).reshape(B * S, n_head * D)
    return alibi_attention_reference(qkv, slopes, B, S, n_head, D)
