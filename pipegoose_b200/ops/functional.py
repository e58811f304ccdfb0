"""Autograd functions of the fast path: each one is a *sub-layer* (several kernels with a
hand-written backward), not a single op, so a transformer block is four autograd nodes and no
elementwise kernel runs outside a GEMM epilogue or a fused normalisation kernel.

Weight gradients are accumulated by the wgrad GEMM epilogue straight into ``param.main_grad``
(fp32, a view into the flat gradient buffer that the fused data-parallel reducer and the fused
ZeRO-1 optimizer consume) when the parameter has one; otherwise they are returned through
autograd like any other gradient, so the same layers work under a stock ``torch.optim``.

Tensor parallelism is expressed through a ``tp`` communicator object (``None`` for TP=1) with
the sequence-parallel contract: activations between sub-layers are sharded along the token
dimension (``[M/T, h]``); column-parallel GEMMs consume an all-gather (fused: AG->GEMM) and
row-parallel GEMMs produce a reduce-scatter (fused: GEMM->RS).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from pipegoose_b200.ops import kernels as K


# lm_head under tensor parallelism through the fused all-gather->GEMM / GEMM->reduce-scatter kernels instead of NCCL
# around a plain GEMM, and LayerNorm backward writing dx straight into the staging slot of the next backward all-gather.
# Covered by tests/test_gpu_multi.py::test_tp2_bloom_matches_single_gpu (2 GPUs) with both;
# PIPEGOOSE_B200_FUSED_LM_HEAD=0 / _LNBWD_TO_STAGE=0 switch them off.
import os as _os

_FUSED_LM_HEAD = _os.environ.get("PIPEGOOSE_B200_FUSED_LM_HEAD", "1") == "1"
_LNBWD_TO_STAGE = _os.environ.get("PIPEGOOSE_B200_LNBWD_TO_STAGE", "1") == "1"
# cross-entropy statistics from the lm_head GEMM's epilogue instead of a pass over the logits: the statistics pass
# never re-reads the [tokens, vocab] logits.  PIPEGOOSE_B200_CE_IN_EPILOGUE=0 restores the separate pass.
_CE_IN_EPILOGUE = _os.environ.get("PIPEGOOSE_B200_CE_IN_EPILOGUE", "1") == "1"


def _main_grad(p: Optional[torch.Tensor]):
    return getattr(p, "main_grad", None) if p is not None else None


def acquire_main_grad(p, will_overwrite: bool):
    """``(main_grad, accumulate)`` for the next gradient contribution to ``p``.

    After a lazy ``zero_grad`` the buffer still holds last step's values (``p._mg_fresh``): the
    first contribution overwrites it (GEMM epilogue without the accumulate flag) or, for
    atomically-built gradients, clears it first."""
    mg = p.main_grad
    if getattr(p, "_mg_fresh", False):
        p._mg_fresh = False
        if will_overwrite:
            return mg, False
        mg.zero_()
    return mg, True


def notify_grad_ready(p):
    """Tell the gradient reducer (if any) that ``p.main_grad`` received a contribution."""
    hook = getattr(p, "_pg_grad_ready", None)
    if hook is not None:
        hook(p)


def _wgrad(dy, x, weight):
    """dW = dy^T x, accumulated into weight.main_grad when present (returns None then)."""
    if _main_grad(weight) is not None:
        mg, accumulate = acquire_main_grad(weight, will_overwrite=True)
        K.gemm_tn(dy, x, accum_into=mg, accumulate=accumulate)
        notify_grad_ready(weight)
        return None
    return K.gemm_tn(dy, x).to(weight.dtype)


def _bgrad(dy, bias):
    if bias is None:
        return None
    if _main_grad(bias) is not None:
        mg, _ = acquire_main_grad(bias, will_overwrite=False)
        K.colsum(dy, accum_into=mg)
        notify_grad_ready(bias)
        return None
    return K.colsum(dy).to(bias.dtype)


def _wgrad_bgrad(dy, x, weight, bias):
    """``(_wgrad(dy, x, weight), _bgrad(dy, bias))``.  When both parameters have main grads, one GEMM computes both:
    the wgrad sums the bias gradient from the ``dy`` tiles it already loads, so ``dy`` is read once."""
    if bias is None or _main_grad(weight) is None or _main_grad(bias) is None:
        return _wgrad(dy, x, weight), _bgrad(dy, bias)
    mg, accumulate = acquire_main_grad(weight, will_overwrite=True)
    mg_b, _ = acquire_main_grad(bias, will_overwrite=False)
    K.gemm_tn(dy, x, accum_into=mg, accumulate=accumulate, bias_grad=mg_b)
    notify_grad_ready(weight)
    notify_grad_ready(bias)
    return None, None


def _ln_bwd(dy, x, gamma, beta, mean, rstd, dx_extra=None, tp=None):
    # Under fused TP the dx of a sub-layer is the dy of the one before it, whose first backward op is an
    # all-gather->GEMM: writing dx straight into that all-gather's staging slot saves a 16 MB copy per sub-layer.
    dx_out = None
    if _LNBWD_TO_STAGE and tp is not None and tp.fused:
        dx_out = tp.ag_input_buffer(x.shape[0], x.shape[1])
    if _main_grad(gamma) is not None and _main_grad(beta) is not None:
        mg_g, _ = acquire_main_grad(gamma, will_overwrite=False)
        mg_b, _ = acquire_main_grad(beta, will_overwrite=False)
        dx, _, _ = K.layernorm_bwd(dy, x, gamma, mean, rstd, dx_extra, mg_g, mg_b, dx_out=dx_out)
        notify_grad_ready(gamma)
        notify_grad_ready(beta)
        return dx, None, None
    return K.layernorm_bwd(dy, x, gamma, mean, rstd, dx_extra, dx_out=dx_out)


def _ln_linear_fwd(x, gamma, beta, weight, bias, eps, tp):
    """LN kernel, then (all-gather ->) GEMM with the bias in the epilogue; returns (y, mean, rstd, ln_full)."""
    stage = tp.ag_input_buffer(x.shape[0], x.shape[1]) if (tp is not None and tp.fused) else None
    ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps, out=stage)
    if tp is not None and tp.fused:
        y, ln_full = tp.ag_gemm(ln, weight, bias)
    else:
        ln_full = tp.all_gather_rows(ln) if tp is not None else ln
        y = K.gemm_nt(ln_full, weight, bias)
    return y, mean, rstd, ln_full


def _ln_linear_bwd(dy, x, gamma, beta, weight, bias, mean, rstd, ln_full, tp, dx_extra=None):
    if tp is not None and tp.fused:
        dln = tp.gemm_rs_nn(dy, weight)
    else:
        dln_full = K.gemm_nn(dy, weight)
        dln = tp.reduce_scatter_rows(dln_full) if tp is not None else dln_full
    dw, db = _wgrad_bgrad(dy, ln_full, weight, bias)
    dx, dgamma, dbeta = _ln_bwd(dln, x, gamma, beta, mean, rstd, dx_extra=dx_extra, tp=tp)
    return dx, dgamma, dbeta, dw, db


def _linear_residual_fwd(a, weight, bias, residual, tp):
    if tp is None:
        return K.gemm_nt(a, weight, bias, residual)
    if tp.fused:
        return tp.gemm_rs(a, weight, bias, residual)
    y = tp.reduce_scatter_rows(K.gemm_nt(a, weight))
    return y + bias + residual if bias is not None else y + residual


def _linear_residual_bwd(dy, a, weight, bias, tp):
    if tp is None:
        dy_full = dy
        da = K.gemm_nn(dy_full, weight)
    elif tp.fused:
        da, dy_full = tp.ag_gemm_nn(dy, weight)
    else:
        dy_full = tp.all_gather_rows(dy)
        da = K.gemm_nn(dy_full, weight)
    if tp is None:
        dw, db = _wgrad_bgrad(dy, a, weight, bias)
        return da, dw, db
    dw = _wgrad(dy_full, a, weight)
    # the bias is replicated across TP ranks: each rank sums its own token shard and the
    # gradient reducer adds the TP group's partial sums (see DataParallel / grad buffer).
    db = _bgrad(dy, bias)
    return da, dw, db


class LayerNormLinear(torch.autograd.Function):
    """``y = Linear(LayerNorm(x))`` — LN kernel, then (all-gather ->) GEMM with the bias in the epilogue.

    Column-parallel under TP: ``x`` is the local token shard ``[M/T, h]``, ``weight`` is
    ``[N/T, h]``, the result is ``[M, N/T]``.
    """

    @staticmethod
    def forward(ctx, x, gamma, beta, weight, bias, eps, tp):
        y, mean, rstd, ln_full = _ln_linear_fwd(x, gamma, beta, weight, bias, eps, tp)
        ctx.save_for_backward(x, gamma, beta, weight, bias, mean, rstd, ln_full)
        ctx.tp = tp
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, weight, bias, mean, rstd, ln_full = ctx.saved_tensors
        dx, dgamma, dbeta, dw, db = _ln_linear_bwd(dy.contiguous(), x, gamma, beta, weight, bias, mean, rstd,
                                                   ln_full, ctx.tp)
        return dx, dgamma, dbeta, dw, db, None, None


class LinearResidual(torch.autograd.Function):
    """``y = a @ W^T + b + residual`` with bias and residual in the GEMM epilogue.

    Row-parallel under TP: ``a`` is ``[M, K/T]``, ``weight`` ``[N, K/T]``; the partial products
    are reduce-scattered over tokens (fused: GEMM->RS) so the result and ``residual`` are the
    local shard ``[M/T, N]``.
    """

    @staticmethod
    def forward(ctx, a, weight, bias, residual, tp):
        y = _linear_residual_fwd(a, weight, bias, residual, tp)
        ctx.save_for_backward(a, weight, bias)
        ctx.tp = tp
        return y

    @staticmethod
    def backward(ctx, dy):
        a, weight, bias = ctx.saved_tensors
        dy = dy.contiguous()
        da, dw, db = _linear_residual_bwd(dy, a, weight, bias, ctx.tp)
        return da, dw, db, dy, None


class AttentionSubLayer(torch.autograd.Function):
    """``y = dense(flash_alibi_attention(qkv(LayerNorm(x)))) + x`` as ONE autograd node (native path):
    LN kernel, (AG->)GEMM+bias, wgmma flash attention, GEMM(->RS)+bias+residual.  The residual-stream
    gradient is added inside the LN backward kernel instead of by an autograd accumulation pass."""

    @staticmethod
    def forward(ctx, x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, tp, seg_start=None):
        from pipegoose_b200.ops import native
        from pipegoose_b200.ops.attention import native_seg_start

        qkv, mean, rstd, ln_full = _ln_linear_fwd(x, gamma, beta, wqkv, bqkv, eps, tp)
        att = torch.empty(B * S, n_head * D, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        seg = native_seg_start(seg_start)
        native().attention_fwd(qkv, slopes, att, lse, B, S, n_head, D, 0.0, seg)
        y = _linear_residual_fwd(att, wd, bd, x, tp)
        ctx.save_for_backward(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, mean, rstd, ln_full, qkv, att, lse, seg)
        ctx.tp = tp
        ctx.dims = (B, S, n_head, D)
        return y

    @staticmethod
    def backward(ctx, dy):
        from pipegoose_b200.ops import native

        x, gamma, beta, wqkv, bqkv, wd, bd, slopes, mean, rstd, ln_full, qkv, att, lse, seg = ctx.saved_tensors
        B, S, n_head, D = ctx.dims
        tp = ctx.tp
        dy = dy.contiguous()
        datt, dwd, dbd = _linear_residual_bwd(dy, att, wd, bd, tp)
        dqkv = torch.empty_like(qkv)
        native().attention_bwd(qkv, slopes, att, lse, datt, dqkv, B, S, n_head, D, 0.0, seg)
        dx, dgamma, dbeta, dwqkv, dbqkv = _ln_linear_bwd(dqkv, x, gamma, beta, wqkv, bqkv, mean, rstd, ln_full, tp,
                                                         dx_extra=dy)
        return dx, dgamma, dbeta, dwqkv, dbqkv, dwd, dbd, None, None, None, None, None, None, None, None


class LayerNormMLP(torch.autograd.Function):
    """``y = fc2(gelu(fc1(LayerNorm(x)))) + b2 + x``: LN kernel, GEMM(+bias+GELU epilogue, keeps the
    pre-activation), GEMM(+bias+residual epilogue).  Backward fuses GELU' into the fc2 dgrad epilogue."""

    @staticmethod
    def forward(ctx, x, gamma, beta, w1, b1, w2, b2, eps, tp):
        stage = tp.ag_input_buffer(x.shape[0], x.shape[1]) if (tp is not None and tp.fused) else None
        ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps, out=stage)
        if tp is not None and tp.fused:
            z_holder = {}
            h1, ln_full = tp.ag_gemm(ln, w1, b1, gelu=True, aux_holder=z_holder)
            z = z_holder["aux"]
            y = tp.gemm_rs(h1, w2, b2, x)
        else:
            ln_full = tp.all_gather_rows(ln) if tp is not None else ln
            z = torch.empty(ln_full.shape[0], w1.shape[0], dtype=ln_full.dtype, device=ln_full.device)
            h1 = K.gemm_nt(ln_full, w1, b1, gelu=True, aux_out=z)
            if tp is None:
                y = K.gemm_nt(h1, w2, b2, x)
            else:
                y = tp.reduce_scatter_rows(K.gemm_nt(h1, w2)) + b2 + x
        ctx.save_for_backward(x, gamma, beta, w1, b1, w2, b2, mean, rstd, ln_full, z, h1)
        ctx.tp = tp
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, w1, b1, w2, b2, mean, rstd, ln_full, z, h1 = ctx.saved_tensors
        tp = ctx.tp
        dy = dy.contiguous()
        if tp is None:
            dy_full = dy
            dz = K.gemm_nn(dy_full, w2, dgelu_aux=z)
        elif tp.fused:
            dz, dy_full = tp.ag_gemm_nn(dy, w2, dgelu_aux=z)
        else:
            dy_full = tp.all_gather_rows(dy)
            dz = K.gemm_nn(dy_full, w2, dgelu_aux=z)
        if tp is None:
            dw2, db2 = _wgrad_bgrad(dy, h1, w2, b2)
        else:
            # row-parallel: the wgrad reads every rank's tokens, the bias sums this rank's shard (see above)
            dw2 = _wgrad(dy_full, h1, w2)
            db2 = _bgrad(dy, b2)
        if tp is not None and tp.fused:
            dln = tp.gemm_rs_nn(dz, w1)
        else:
            dln_full = K.gemm_nn(dz, w1)
            dln = tp.reduce_scatter_rows(dln_full) if tp is not None else dln_full
        dw1, db1 = _wgrad_bgrad(dz, ln_full, w1, b1)
        # residual gradient (dy) is added inside the LN backward kernel
        dx, dgamma, dbeta = _ln_bwd(dln, x, gamma, beta, mean, rstd, dx_extra=dy, tp=tp)
        return dx, dgamma, dbeta, dw1, db1, dw2, db2, None, None


# ----------------------------------------------------------------------------------------------
# FP8 sub-layers (BloomConfig.fp8): the four linear layers of a block on the FP8 GEMM, everything else as above.
# Per-tensor current scaling (ops.kernels.fp8_quantize): activations and weights e4m3, gradients e5m2.  FP8 wgmma reads
# both operands K-major, so every cast also writes the transposed codes and every product is the forward (NT) layout:
#   forward  Y  = X  · Wᵀ : X codes [M, K],  W codes [N, K]
#   dgrad    dX = dY · W  : dY codes [M, N], Wᵀ codes [K, N]
#   wgrad    dW = dYᵀ · X : dYᵀ codes [N, M], Xᵀ codes [K, M]
# The forward saves Wᵀ codes and the GEMM inputs' transposed codes (half the bytes of the bf16 inputs) for backward.
# Bias gradients are the fp32 column sums of the bf16 dY, summed by its cast; wgrads go through the fp32 TMA epilogue
# into main_grad with the same acquire_main_grad / notify_grad_ready protocol as the bf16 layers.
# ----------------------------------------------------------------------------------------------
def _fp8_cast_grad(dy, bias):
    """e5m2 codes of ``dy`` and of ``dyᵀ``, ``scale_inv``, and the bias gradient: added into ``bias.main_grad`` by the
    cast (then ``None``) or returned."""
    mg = None
    if bias is not None:
        if _main_grad(bias) is not None:
            mg, _ = acquire_main_grad(bias, will_overwrite=False)
        else:
            mg = torch.zeros(dy.shape[1], dtype=torch.float32, device=dy.device)
    c, ct, s = K.fp8_quantize(dy, "e5m2", transpose=True, colsum_into=mg)
    db = None
    if bias is not None:
        if _main_grad(bias) is not None:
            notify_grad_ready(bias)
        else:
            db = mg.to(bias.dtype)
    return c, ct, s, db


def _fp8_wgrad(dy_t, s_dy, x_t, s_x, weight):
    """``dW = dyᵀ x`` from the transposed codes, into ``weight.main_grad`` (then ``None``) or returned."""
    mg = _main_grad(weight)
    if mg is not None and K.grad_rs_for(mg) is None:
        mg, accumulate = acquire_main_grad(weight, will_overwrite=True)
        K.gemm_fp8(dy_t, x_t, s_dy, s_x, accum_into=mg, accumulate=accumulate)
        notify_grad_ready(weight)
        return None
    g = torch.empty(dy_t.shape[0], x_t.shape[0], dtype=torch.float32, device=dy_t.device)
    K.gemm_fp8(dy_t, x_t, s_dy, s_x, accum_into=g)
    if mg is None:
        return g.to(weight.dtype)
    # a main grad reduce-scattered in-kernel (ZeRO-1): the FP8 GEMM has no such epilogue, the fold kernel adds it
    mg, accumulate = acquire_main_grad(weight, will_overwrite=True)
    K.accumulate_grad(g, mg, accumulate)
    notify_grad_ready(weight)
    return None


def _fp8_cast(x):
    """e4m3 codes, transposed codes and ``scale_inv`` of an activation or weight."""
    return K.fp8_quantize(x.contiguous(), "e4m3", transpose=True)


def _attention_width(D):
    """``(DP, softmax scale)`` of the flash kernel for head size ``D``: D itself (scale 0: the kernel's 1/sqrt(D)), or
    heads zero-padded to DP with the true width's scale (``ops.attention._AlibiAttentionPadded``, e.g. D = 80)."""
    from pipegoose_b200.ops.attention import _native_attention_available, padded_head_dim

    if _native_attention_available(D):
        return D, 0.0
    return padded_head_dim(D), 1.0 / math.sqrt(D)


class AttentionSubLayerFP8(torch.autograd.Function):
    """:class:`AttentionSubLayer` (no tensor parallelism) with qkv and dense on the FP8 GEMM.  Head sizes without a
    flash tile of their own (D = 80) run padded, as :func:`ops.attention.alibi_attention` does."""

    @staticmethod
    def forward(ctx, x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, seg_start=None):
        from pipegoose_b200.ops import native
        from pipegoose_b200.ops.attention import native_seg_start, pad_heads, unpad_heads

        DP, scale = _attention_width(D)
        ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps)
        ln_c, ln_t, s_ln = _fp8_cast(ln)
        del ln
        wq_c, wq_t, s_wq = _fp8_cast(wqkv)
        qkv = K.gemm_fp8(ln_c, wq_c, s_ln, s_wq, bias=bqkv)
        del ln_c, wq_c
        qkv = pad_heads(qkv, n_head, 3, D, DP).contiguous()
        att_p = torch.empty(B * S, n_head * DP, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, n_head, S, dtype=torch.float32, device=qkv.device)
        seg = native_seg_start(seg_start)
        native().attention_fwd(qkv, slopes, att_p, lse, B, S, n_head, DP, scale, seg)
        att_c, att_t, s_att = _fp8_cast(unpad_heads(att_p, n_head, 1, D, DP))
        wd_c, wd_t, s_wd = _fp8_cast(wd)
        y = K.gemm_fp8(att_c, wd_c, s_att, s_wd, bias=bd, residual=x)
        ctx.save_for_backward(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, mean, rstd, ln_t, s_ln, wq_t, s_wq, qkv,
                              att_p, lse, att_t, s_att, wd_t, s_wd, seg)
        ctx.dims = (B, S, n_head, D, DP, scale)
        return y

    @staticmethod
    def backward(ctx, dy):
        from pipegoose_b200.ops import native
        from pipegoose_b200.ops.attention import pad_heads, unpad_heads

        (x, gamma, beta, wqkv, bqkv, wd, bd, slopes, mean, rstd, ln_t, s_ln, wq_t, s_wq, qkv, att_p, lse, att_t, s_att,
         wd_t, s_wd, seg) = ctx.saved_tensors
        B, S, n_head, D, DP, scale = ctx.dims
        dy = dy.contiguous()
        dy_c, dy_t, s_dy, dbd = _fp8_cast_grad(dy, bd)
        datt = K.gemm_fp8(dy_c, wd_t, s_dy, s_wd)
        dwd = _fp8_wgrad(dy_t, s_dy, att_t, s_att, wd)
        del dy_c, dy_t
        datt = pad_heads(datt, n_head, 1, D, DP).contiguous()
        dqkv = torch.empty_like(qkv)
        native().attention_bwd(qkv, slopes, att_p, lse, datt, dqkv, B, S, n_head, DP, scale, seg)
        del datt
        dqkv = unpad_heads(dqkv, n_head, 3, D, DP).contiguous()
        dq_c, dq_t, s_dq, dbqkv = _fp8_cast_grad(dqkv, bqkv)
        del dqkv
        dln = K.gemm_fp8(dq_c, wq_t, s_dq, s_wq)
        dwqkv = _fp8_wgrad(dq_t, s_dq, ln_t, s_ln, wqkv)
        dx, dgamma, dbeta = _ln_bwd(dln, x, gamma, beta, mean, rstd, dx_extra=dy)
        return dx, dgamma, dbeta, dwqkv, dbqkv, dwd, dbd, None, None, None, None, None, None, None


class LayerNormMLPFP8(torch.autograd.Function):
    """:class:`LayerNormMLP` (no tensor parallelism) with fc1 and fc2 on the FP8 GEMM: GELU and its pre-activation in
    the fc1 epilogue, GELU' on the bf16 pre-activation in the fc2 dgrad epilogue."""

    @staticmethod
    def forward(ctx, x, gamma, beta, w1, b1, w2, b2, eps):
        ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps)
        ln_c, ln_t, s_ln = _fp8_cast(ln)
        del ln
        w1_c, w1_t, s_w1 = _fp8_cast(w1)
        z = torch.empty(x.shape[0], w1.shape[0], dtype=x.dtype, device=x.device)
        h1 = K.gemm_fp8(ln_c, w1_c, s_ln, s_w1, bias=b1, gelu=True, aux_out=z)
        del ln_c, w1_c
        h1_c, h1_t, s_h1 = _fp8_cast(h1)
        del h1
        w2_c, w2_t, s_w2 = _fp8_cast(w2)
        y = K.gemm_fp8(h1_c, w2_c, s_h1, s_w2, bias=b2, residual=x)
        ctx.save_for_backward(x, gamma, beta, w1, b1, w2, b2, mean, rstd, ln_t, s_ln, w1_t, s_w1, z, h1_t, s_h1, w2_t,
                              s_w2)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, w1, b1, w2, b2, mean, rstd, ln_t, s_ln, w1_t, s_w1, z, h1_t, s_h1, w2_t, s_w2 = ctx.saved_tensors
        dy = dy.contiguous()
        dy_c, dy_t, s_dy, db2 = _fp8_cast_grad(dy, b2)
        dz = K.gemm_fp8(dy_c, w2_t, s_dy, s_w2, dgelu_aux=z)
        dw2 = _fp8_wgrad(dy_t, s_dy, h1_t, s_h1, w2)
        del dy_c, dy_t
        dz_c, dz_t, s_dz, db1 = _fp8_cast_grad(dz, b1)
        del dz
        dln = K.gemm_fp8(dz_c, w1_t, s_dz, s_w1)
        dw1 = _fp8_wgrad(dz_t, s_dz, ln_t, s_ln, w1)
        dx, dgamma, dbeta = _ln_bwd(dln, x, gamma, beta, mean, rstd, dx_extra=dy)
        return dx, dgamma, dbeta, dw1, db1, dw2, db2, None


def _fp8_check(x, *weights):
    """The FP8 sub-layers run on the sm_90a kernels only, at shapes the FP8 GEMM takes."""
    from pipegoose_b200.ops import use_native

    if not use_native(x, *weights):
        raise ValueError("fp8=True runs on the native path only (CUDA bf16 model and inputs); this model does not")
    dims = [x.shape[0]] + [d for w in weights for d in w.shape]
    if any(d % 16 for d in dims):
        raise ValueError(f"fp8=True needs the token count and every linear layer's width to be multiples of 16, got "
                         f"{x.shape[0]} tokens and weights {[tuple(w.shape) for w in weights]}")


class Linear(torch.autograd.Function):
    """``y = x @ W^T + b`` for any leading shape: wgmma GEMM (bias in the epilogue), dgrad and wgrad
    GEMMs in backward.  Used by the reference-compatible Column/RowParallelLinear layers."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        y = K.gemm_nt(x2, weight, bias)
        ctx.save_for_backward(x2, weight, bias)
        ctx.shape = shape
        return y.view(*shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, weight, bias = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dx = K.gemm_nn(dy2, weight).view(ctx.shape) if ctx.needs_input_grad[0] else None
        dw = _wgrad(dy2, x2, weight) if ctx.needs_input_grad[1] else None
        db = _bgrad(dy2, bias) if bias is not None and ctx.needs_input_grad[2] else None
        return dx, dw, db


def linear(x, weight, bias=None):
    """Drop-in for ``F.linear`` that runs on the sm_90a GEMM when ``x`` is a CUDA bf16 tensor."""
    from pipegoose_b200.ops import use_native

    if use_native(x, weight) and weight.shape[0] % 8 == 0 and weight.shape[1] % 8 == 0:
        return Linear.apply(x, weight, bias)
    return torch.nn.functional.linear(x, weight, bias)


class MLPResidual(torch.autograd.Function):
    """``y = fc2(gelu(fc1(x))) + b2 + residual`` (no LayerNorm, no TP): the dense MLP used as an MoE
    expert and behind HF's ``mlp(hidden_states, residual)`` signature."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, residual):
        z = torch.empty(x.shape[0], w1.shape[0], dtype=x.dtype, device=x.device)
        h1 = K.gemm_nt(x, w1, b1, gelu=True, aux_out=z)
        y = K.gemm_nt(h1, w2, b2, residual)
        ctx.save_for_backward(x, w1, b1, w2, b2, z, h1)
        ctx.has_residual = residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w1, b1, w2, b2, z, h1 = ctx.saved_tensors
        dy = dy.contiguous()
        dz = K.gemm_nn(dy, w2, dgelu_aux=z)
        dw2 = _wgrad(dy, h1, w2)
        db2 = _bgrad(dy, b2)
        dx = K.gemm_nn(dz, w1)
        dw1 = _wgrad(dz, x, w1)
        db1 = _bgrad(dz, b1)
        return dx, dw1, db1, dw2, db2, (dy if ctx.has_residual else None)


class EmbeddingLayerNorm(torch.autograd.Function):
    """``LayerNorm(table[ids])`` in one kernel (vocab-parallel aware); backward scatter-adds into
    the table's fp32 main grad."""

    @staticmethod
    def forward(ctx, ids, table, gamma, beta, eps, vocab_start, tp):
        vocab_end = vocab_start + table.shape[0]
        flat = ids.reshape(-1)
        if tp is None:
            y, mean, rstd = K.layernorm_fwd(table, gamma, beta, eps, ids=flat, vocab_start=vocab_start, vocab_end=vocab_end)
            e = None
        else:
            part, _, _ = K.layernorm_fwd(table, gamma, beta, eps, ids=flat, vocab_start=vocab_start,
                                         vocab_end=vocab_end, apply_ln=False)
            e = tp.reduce_scatter_rows(part.contiguous())  # [M/T, h] complete embeddings of the local tokens
            y, mean, rstd = K.layernorm_fwd(e, gamma, beta, eps)
        ctx.save_for_backward(flat, table, gamma, beta, mean, rstd, e if e is not None else torch.empty(0))
        ctx.tp = tp
        ctx.eps = eps
        ctx.vocab_start = vocab_start
        return y

    @staticmethod
    def backward(ctx, dy):
        flat, table, gamma, beta, mean, rstd, e = ctx.saved_tensors
        tp = ctx.tp
        vocab_start = ctx.vocab_start
        vocab_end = vocab_start + table.shape[0]
        dy = dy.contiguous()
        if tp is None:
            e, _, _ = K.layernorm_fwd(table, gamma, beta, ctx.eps, ids=flat, vocab_start=vocab_start,
                                      vocab_end=vocab_end, apply_ln=False)
        de, dgamma, dbeta = _ln_bwd(dy, e, gamma, beta, mean, rstd)
        de_full = tp.all_gather_rows(de) if tp is not None else de
        mg = acquire_main_grad(table, will_overwrite=False)[0] if _main_grad(table) is not None else None
        dtable = K.embedding_bwd(de_full, flat, table.shape[0], vocab_start, vocab_end, accum_into=mg)
        if mg is not None:
            notify_grad_ready(table)
        return None, dtable, dgamma, dbeta, None, None, None


class EmbeddingPositions(torch.autograd.Function):
    """``table[ids] + positions[pos]`` for models with learned position embeddings (GPT-2), vocab-parallel and
    sequence-parallel aware: under TP every rank gathers the rows of its vocabulary slice for ALL tokens, the partial
    results are reduce-scattered over the token dimension, and the position rows of the LOCAL tokens are added.  The
    backward scatter-adds into the table's fp32 main grad like :class:`EmbeddingLayerNorm`; the position-table gradient
    is a partial sum over this rank's tokens (the parameter is tagged ``tp_partial_grad``).

    ``position_ids`` (``[B, S]``, packed sequences): the position of every token, flattened like the tokens; the local
    rows' slice of it replaces ``arange(S)``."""

    @staticmethod
    def forward(ctx, ids, table, positions, vocab_start, tp, position_ids=None):
        vocab_end = vocab_start + table.shape[0]
        flat = ids.reshape(-1)
        seq = ids.shape[-1]
        dummy = positions[0]  # gamma / beta arguments of the gather kernel (unused with apply_ln=False)
        part, _, _ = K.layernorm_fwd(table, dummy, dummy, 0.0, ids=flat, vocab_start=vocab_start, vocab_end=vocab_end,
                                     apply_ln=False)
        e = tp.reduce_scatter_rows(part.contiguous()) if tp is not None else part
        rows = e.shape[0]
        first = tp.rank * rows if tp is not None else 0
        if position_ids is None:
            pos = (torch.arange(rows, device=e.device) + first) % seq
        else:
            pos = position_ids.reshape(-1)[first:first + rows].to(device=e.device, dtype=torch.long)
        ctx.save_for_backward(flat, table, positions, pos)
        ctx.tp = tp
        ctx.vocab_start = vocab_start
        return e + positions.index_select(0, pos)

    @staticmethod
    def backward(ctx, dy):
        flat, table, positions, pos = ctx.saved_tensors
        tp, vocab_start = ctx.tp, ctx.vocab_start
        vocab_end = vocab_start + table.shape[0]
        dy = dy.contiguous()
        dpos = torch.zeros(positions.shape, dtype=torch.float32, device=dy.device).index_add_(0, pos, dy.float())
        mg_pos = _main_grad(positions)
        if mg_pos is not None:
            acc, accumulate = acquire_main_grad(positions, will_overwrite=True)
            K.accumulate_grad(dpos, acc, accumulate)   # (goes through the in-kernel reduce-scatter when acc is in one)
            notify_grad_ready(positions)
            dpos = None
        else:
            dpos = dpos.to(positions.dtype)
        de_full = tp.all_gather_rows(dy) if tp is not None else dy
        mg = acquire_main_grad(table, will_overwrite=False)[0] if _main_grad(table) is not None else None
        dtable = K.embedding_bwd(de_full, flat, table.shape[0], vocab_start, vocab_end, accum_into=mg)
        if mg is not None:
            notify_grad_ready(table)
        return None, dtable, dpos, None, None, None


class LMHeadCrossEntropy(torch.autograd.Function):
    """``mean CE(LayerNorm(x) @ table^T, labels)`` with a vocab-parallel softmax.

    The logits GEMM writes bf16 logits once; one stats kernel + one finalize kernel turn them into
    the loss and, in place, ``dlogits`` (already scaled by 1/num_tokens), which feed the dgrad and
    wgrad GEMMs directly.  Across TP ranks only ``[M, 3]`` floats are exchanged (max, sum-exp,
    target logit) instead of the reference's all-gather of ``[M, V]`` logits.
    """

    @staticmethod
    def forward(ctx, x, gamma, beta, table, labels, eps, vocab_start, ignore_index, tp, vocab_size=None):
        from pipegoose_b200.ops import use_native

        fused = tp is not None and tp.fused and _FUSED_LM_HEAD
        v_local = table.shape[0]
        real = v_local if vocab_size is None else min(max(vocab_size - vocab_start, 0), v_local)
        rows_full = x.shape[0] * (tp.size if tp is not None else 1)
        # The logits GEMM's epilogue also emits the online-softmax partials (max, sum exp) of every half tile it holds in
        # registers: the cross entropy's statistics pass over the [tokens, vocab] logits disappears
        part = K.ce_partials_buffer(rows_full, v_local, x.device) if (_CE_IN_EPILOGUE and use_native(x, table)) else None
        extra = {"ce_part": part.data_ptr(), "ce_valid": real} if part is not None else None
        if fused:
            # all-gather -> GEMM like every other column-parallel linear (LN writes into the gather staging buffer)
            stage = tp.ag_input_buffer(x.shape[0], x.shape[1])
            ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps, out=stage)
            logits, ln_full = tp.ag_gemm(ln, table, extra=extra)
        else:
            ln, mean, rstd = K.layernorm_fwd(x, gamma, beta, eps)
            ln_full = tp.all_gather_rows(ln) if tp is not None else ln
            logits = K.gemm_nt(ln_full, table, **({"ag": extra} if extra else {}))  # [M, V/T]
        if real < logits.shape[1]:
            # rows the table was zero-padded with (vocabulary made divisible by the group size) are not classes: their
            # logits leave the softmax (-inf: exp 0, gradient 0).  Only the last shard(s) have any; no-op otherwise.
            logits[:, real:] = float("-inf")
        tgt = labels.reshape(-1)
        stats = K.ce_stats_from_partials(part, logits, tgt, vocab_start) if part is not None \
            else K.ce_local_stats(logits, tgt, vocab_start)
        if tp is not None:
            gstats = K.ce_combine_stats(tp.all_gather_stack(stats))
        else:
            gstats = stats
        n_valid = (tgt != ignore_index).sum().clamp(min=1).to(torch.float32)
        loss_rows = K.ce_finalize(logits, tgt, gstats, vocab_start, None, ignore_index, write_grad=False)
        loss = loss_rows.sum() / n_valid
        ctx.save_for_backward(x, gamma, beta, table, mean, rstd, ln_full, logits, n_valid, tgt, gstats)
        ctx.tp = tp
        ctx.vocab_start = vocab_start
        ctx.ignore_index = ignore_index
        return loss

    @staticmethod
    def backward(ctx, dloss):
        x, gamma, beta, table, mean, rstd, ln_full, logits, n_valid, tgt, gstats = ctx.saved_tensors
        tp = ctx.tp
        # dlogits = (softmax - onehot) * dloss / n_valid, written over the logits in one pass; the
        # scale stays on the device (no host sync)
        scale = (dloss.float() / n_valid).reshape(1)
        K.ce_finalize(logits, tgt, gstats, ctx.vocab_start, scale, ctx.ignore_index, write_grad=True)
        dlogits = logits
        if tp is not None and tp.fused and _FUSED_LM_HEAD:
            dln = tp.gemm_rs_nn(dlogits, table)  # GEMM -> reduce-scatter over NVLink, no [M, h] NCCL round trip
        else:
            dln_full = K.gemm_nn(dlogits, table)
            dln = tp.reduce_scatter_rows(dln_full) if tp is not None else dln_full
        dtable = _wgrad(dlogits, ln_full, table)
        dx, dgamma, dbeta = _ln_bwd(dln, x, gamma, beta, mean, rstd)
        return dx, dgamma, dbeta, dtable, None, None, None, None, None, None


def layernorm_linear(x, gamma, beta, weight, bias, eps=1e-5, tp=None):
    return LayerNormLinear.apply(x, gamma, beta, weight, bias, eps, tp)


def attention_sublayer(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, tp=None, seg_start=None):
    """LN -> QKV -> causal ALiBi attention -> dense + residual (``x`` is the residual stream).  ``seg_start``: document
    starts of packed rows (``ops.attention``), the same full-length tensor on every tensor-parallel rank: attention runs
    on the all-gathered tokens."""
    from pipegoose_b200.ops import use_native
    from pipegoose_b200.ops.attention import _native_attention_available, alibi_attention

    if use_native(x, wqkv) and _native_attention_available(D):
        return AttentionSubLayer.apply(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, tp, seg_start)
    qkv = LayerNormLinear.apply(x, gamma, beta, wqkv, bqkv, eps, tp)
    att = alibi_attention(qkv, slopes, B, S, n_head, D, seg_start=seg_start)
    return LinearResidual.apply(att, wd, bd, x, tp)


def attention_sublayer_fp8(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, seg_start=None):
    """:func:`attention_sublayer` with the qkv and dense GEMMs in FP8 (no tensor parallelism)."""
    _fp8_check(x, wqkv, wd)
    if _attention_width(D)[0] == 0 or D % 8:
        raise ValueError(f"fp8=True needs a head size the flash attention kernel runs (natively or zero-padded: "
                         f"D <= 128, a multiple of 8), got {D}")
    return AttentionSubLayerFP8.apply(x, gamma, beta, wqkv, bqkv, wd, bd, slopes, eps, B, S, n_head, D, seg_start)


def layernorm_mlp_fp8(x, gamma, beta, w1, b1, w2, b2, eps=1e-5):
    """:func:`layernorm_mlp` with fc1 and fc2 in FP8 (no tensor parallelism)."""
    _fp8_check(x, w1, w2)
    return LayerNormMLPFP8.apply(x, gamma, beta, w1, b1, w2, b2, eps)

def linear_residual(a, weight, bias, residual, tp=None):
    return LinearResidual.apply(a, weight, bias, residual, tp)


def layernorm_mlp(x, gamma, beta, w1, b1, w2, b2, eps=1e-5, tp=None):
    return LayerNormMLP.apply(x, gamma, beta, w1, b1, w2, b2, eps, tp)


def mlp_residual(x, w1, b1, w2, b2, residual=None):
    return MLPResidual.apply(x, w1, b1, w2, b2, residual)


def embedding_layernorm(ids, table, gamma, beta, eps=1e-5, vocab_start=0, tp=None):
    return EmbeddingLayerNorm.apply(ids, table, gamma, beta, eps, vocab_start, tp)


def embedding_positions(ids, table, positions, vocab_start=0, tp=None, position_ids=None):
    return EmbeddingPositions.apply(ids, table, positions, vocab_start, tp, position_ids)


def lm_head_cross_entropy(x, gamma, beta, table, labels, eps=1e-5, vocab_start=0, ignore_index=-100, tp=None,
                          vocab_size=None):
    """``vocab_size``: the true (global) vocabulary size when the table was padded for tensor parallelism."""
    return LMHeadCrossEntropy.apply(x, gamma, beta, table, labels, eps, vocab_start, ignore_index, tp, vocab_size)
