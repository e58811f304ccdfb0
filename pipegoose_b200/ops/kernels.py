"""Thin functional wrappers over the native kernels with PyTorch reference fallbacks.

Each wrapper has one contract and two implementations: the sm_90a kernel (CUDA bf16 tensors,
mandatory on GPU machines) and plain PyTorch math (CPU / fp32, used by the gloo unit tests and
as the numerics oracle in the GPU tests).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from pipegoose_b200.ops import native, use_native

EPI_BIAS, EPI_GELU, EPI_RESIDUAL, EPI_OUT_F32, EPI_ACCUM, EPI_DGELU, EPI_SCATTER = 1, 2, 4, 8, 16, 32, 64


# ----------------------------------------------------------------------------------------------
# in-kernel data-parallel gradient reduce-scatter (ZeRO-1): address ranges of flat fp32 gradient buffers whose
# contributions are added straight into the OWNER rank's buffer by the producing kernel (csrc/grad_rs.cuh).  Every
# gradient writer below looks its destination up here, so a writer can never bypass the reduction by accident.
# ----------------------------------------------------------------------------------------------
_GRAD_RS_REGIONS = []   # [(first byte, end byte, descriptor dict for the kernels, engine)]


def register_grad_rs(begin: int, end: int, desc: dict, engine) -> None:
    import weakref

    unregister_grad_rs(engine)
    _GRAD_RS_REGIONS.append((begin, end, desc, weakref.ref(engine)))   # (weak: a dropped engine unregisters itself)


def unregister_grad_rs(engine) -> None:
    _GRAD_RS_REGIONS[:] = [r for r in _GRAD_RS_REGIONS if r[3]() is not None and r[3]() is not engine]


def grad_rs_for(t: Optional[torch.Tensor]):
    """The reduce-scatter descriptor if ``t`` (a view of a flat gradient buffer) lies in a registered region."""
    if not _GRAD_RS_REGIONS or t is None or not t.is_cuda:
        return None
    ptr = t.data_ptr()
    for begin, end, desc, ref in _GRAD_RS_REGIONS:
        engine = ref()
        if engine is not None and begin <= ptr < end:
            engine.inline_dirty = True
            return desc
    return None


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    """Bloom's GELU (tanh approximation; transformers BloomGelu)."""
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1.0 + 0.044715 * x * x)))


def gelu_tanh_grad(x: torch.Tensor) -> torch.Tensor:
    t = torch.tanh(0.79788456 * x * (1.0 + 0.044715 * x * x))
    return 0.5 * x * ((1 - t * t) * (0.79788456 + 0.1070322243 * x * x)) + 0.5 * (1 + t)


# ----------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------
def gemm_nt(x, w, bias=None, residual=None, gelu=False, aux_out=None, out=None, **kw):
    """``out[M,N] = epi(x[M,K] @ w[N,K]^T)``: bias, tanh-GELU (pre-activation into ``aux_out``), residual."""
    if use_native(x, w):
        M, N = x.shape[0], w.shape[0]
        if out is None:
            out = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
        flags = EPI_GELU if gelu else 0
        native().gemm(x, w, out, False, False, bias, residual, aux_out if gelu else None, flags, **kw)
        return out
    y = x @ w.t()
    if bias is not None:
        y = y + bias
    if gelu:
        if aux_out is not None:
            aux_out.copy_(y)
        y = gelu_tanh(y)
    if residual is not None:
        y = y + residual
    if out is not None:
        out.copy_(y)
        return out
    return y


def gemm_nn(dy, w, dgelu_aux=None, out=None, **kw):
    """``out[M,K] = dy[M,N] @ w[N,K]`` (dgrad); optional ``* gelu'(aux)`` epilogue."""
    if use_native(dy, w):
        M, K = dy.shape[0], w.shape[1]
        if out is None:
            out = torch.empty(M, K, dtype=torch.bfloat16, device=dy.device)
        flags = EPI_DGELU if dgelu_aux is not None else 0
        native().gemm(dy, w, out, False, True, None, None, dgelu_aux, flags, **kw)
        return out
    y = dy @ w
    if dgelu_aux is not None:
        y = y * gelu_tanh_grad(dgelu_aux.float()).to(y.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def gemm_tn(dy, x, accum_into: Optional[torch.Tensor] = None, accumulate: bool = True,
            bias_grad: Optional[torch.Tensor] = None, **kw):
    """``dW[N,K] = dy[M,N]^T @ x[M,K]`` (wgrad).  With ``accum_into`` (fp32 main grad) the product is
    accumulated in place by the GEMM epilogue and ``None`` is returned.  ``bias_grad`` (fp32 ``[N]``, with
    ``accum_into``): the column sums of ``dy`` are added into it by the same kernel (``colsum(dy, bias_grad)``)."""
    assert bias_grad is None or accum_into is not None, "bias_grad needs accum_into"
    if use_native(dy, x):
        N, K = dy.shape[1], x.shape[1]
        if accum_into is not None:
            rs = grad_rs_for(accum_into)
            if rs is not None:
                # wgrad -> reduce-scatter in one kernel: the epilogue adds every tile into its owner's gradient buffer
                kw = dict(kw)
                kw["ag"] = dict(kw.get("ag") or {}, grad_rs=rs)
                accumulate = True
            native().gemm(dy, x, accum_into.view(N, K), True, True, None, None, None,
                          EPI_ACCUM if accumulate else 0, bias_grad=bias_grad, **kw)
            return None
        out = torch.empty(N, K, dtype=torch.bfloat16, device=dy.device)
        native().gemm(dy, x, out, True, True, None, None, None, 0, **kw)
        return out
    if bias_grad is not None:
        colsum(dy, accum_into=bias_grad)
    g = dy.t() @ x
    if accum_into is not None:
        if accumulate:
            accum_into.view_as(g).add_(g.to(accum_into.dtype))
        else:
            accum_into.view_as(g).copy_(g.to(accum_into.dtype))
        return None
    return g


# ----------------------------------------------------------------------------------------------
# FP8 (per-tensor current scaling) for the FP8 linear layers
# ----------------------------------------------------------------------------------------------
FP8_FORMATS = {"e4m3": (torch.float8_e4m3fn, 448.0), "e5m2": (torch.float8_e5m2, 57344.0)}


def fp8_quantize_reference(x: torch.Tensor, fmt: str):
    """The FP8 cast's definition (and the oracle of its kernel): ``x`` -> (codes of ``x``'s shape, fp32 ``scale_inv``
    of shape ``[1]``) with ``x ~ codes * scale_inv``.  In fp32, with IEEE division (tensor by tensor: torch computes
    ``scalar / tensor`` as a reciprocal product):

    * ``amax = max |x|``, ``fmax`` = 448 (``"e4m3"``) or 57344 (``"e5m2"``);
    * ``scale = min(fmax / amax, FLT_MAX)``, 1 when ``amax == 0``; ``code = rn(clamp(x * scale, -fmax, fmax))``;
    * ``scale_inv = amax / fmax``, 1 when ``amax == 0``, NaN when ``amax`` is not finite (an inf or NaN in a gradient
      must not turn into finite codes)."""
    dtype, fmax = FP8_FORMATS[fmt]
    xf = x.float()
    amax = xf.abs().amax().reshape(1) if xf.numel() else torch.zeros(1, device=x.device)
    m = torch.full_like(amax, fmax)
    zero = amax == 0
    scale = torch.where(zero, torch.ones_like(amax), torch.fmin(m / amax, torch.full_like(amax, torch.finfo(torch.float32).max)))
    codes = torch.clamp(xf * scale, -fmax, fmax).to(dtype)
    scale_inv = torch.where(zero, torch.ones_like(amax), amax / m)
    scale_inv = torch.where(torch.isfinite(amax), scale_inv, torch.full_like(amax, float("nan")))
    return codes, scale_inv


def fp8_quantize(x: torch.Tensor, fmt: str, codes: bool = True, transpose: bool = False,
                 colsum_into: Optional[torch.Tensor] = None):
    """Per-tensor FP8 cast of a contiguous bf16 CUDA matrix ``x [R, C]`` (``C % 8 == 0``) in two kernels (amax, then
    cast), with no host sync.  Returns ``(codes [R, C] or None, codes_t [C, R] or None, scale_inv [1] fp32)`` in the
    format of :func:`fp8_quantize_reference`, bit for bit.  ``colsum_into`` (fp32 ``[C]``): the column sums of ``x``
    (bf16 values, fp32 sums) are added into it by the same pass."""
    dtype, _ = FP8_FORMATS[fmt]
    R, C = x.shape
    ws = torch.empty(2, dtype=torch.float32, device=x.device)   # [amax, scale_inv]
    c = torch.empty(R, C, dtype=dtype, device=x.device) if codes else None
    ct = torch.empty(C, R, dtype=dtype, device=x.device) if transpose else None
    scale_inv = ws[1:]
    native().fp8_quantize(x, fmt == "e5m2", ws, codes=c, codes_t=ct, scale_inv=scale_inv, colsum=colsum_into)
    return c, ct, scale_inv


def gemm_fp8(a, b, a_scale_inv, b_scale_inv, bias=None, residual=None, gelu=False, aux_out=None, dgelu_aux=None,
             accum_into: Optional[torch.Tensor] = None, accumulate: bool = False, out=None, block_n: int = 0,
             k_splits: int = 0):
    """``out[M, N] = epi(a_scale_inv * b_scale_inv * (a[M, K] @ b[N, K]^T))`` on FP8 codes (``a`` e4m3 or e5m2, ``b``
    e4m3, both K-major, ``K % 16 == 0``).  bf16 out with bias, tanh-GELU (pre-activation into ``aux_out``), residual
    or ``* gelu'(dgelu_aux)``; or, with ``accum_into`` (fp32 ``[M, N]``), overwritten (``accumulate=False``) or added
    into.  There is no fallback: FP8 runs on the sm_90a kernel only."""
    M, N = a.shape[0], b.shape[0]
    if accum_into is not None:
        native().gemm_fp8(a, b, a_scale_inv, b_scale_inv, accum_into.view(M, N), accumulate=accumulate,
                          block_n=block_n, k_splits=k_splits)
        return None
    if out is None:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=a.device)
    aux = aux_out if gelu else dgelu_aux
    native().gemm_fp8(a, b, a_scale_inv, b_scale_inv, out, bias=bias, residual=residual, aux=aux, gelu=gelu,
                      dgelu=dgelu_aux is not None, block_n=block_n, k_splits=k_splits)
    return out


def colsum(dy, accum_into: Optional[torch.Tensor] = None):
    """Bias gradient: column sums of ``dy`` (accumulated into the fp32 main grad when given)."""
    if use_native(dy):
        if accum_into is not None:
            native().colsum(dy, accum_into)
            return None
        out = torch.zeros(dy.shape[1], dtype=torch.float32, device=dy.device)
        native().colsum(dy, out)
        return out.to(dy.dtype)
    g = dy.float().sum(0)
    if accum_into is not None:
        accum_into.add_(g.to(accum_into.dtype))
        return None
    return g.to(dy.dtype)


def accumulate_grad(grad, main_grad, accumulate: bool = True, scale: float = 1.0):
    """``main_grad (+)= scale * grad``: cast (bf16 -> fp32), scale and accumulate in one pass."""
    rs = grad_rs_for(main_grad)
    if rs is not None:
        # the destination is reduce-scattered in-kernel: the contribution goes to the owners of its slices
        src = grad if grad.dtype in (torch.bfloat16, torch.float32) else grad.float()
        native().grad_rs_accum(src.contiguous().view(-1), main_grad.view(-1), scale, rs)
        return
    if use_native(grad) and main_grad.dtype == torch.float32 and grad.is_contiguous():
        native().accum_bf16_to_f32(grad, main_grad, scale, accumulate)
        return
    g = grad.to(main_grad.dtype) * scale if scale != 1.0 else grad.to(main_grad.dtype)
    if accumulate:
        main_grad.add_(g.view_as(main_grad))
    else:
        main_grad.copy_(g.view_as(main_grad))


# ----------------------------------------------------------------------------------------------
# LayerNorm (+ fused embedding gather)
# ----------------------------------------------------------------------------------------------
def layernorm_fwd(x, gamma, beta, eps, ids=None, vocab_start=0, vocab_end=0, apply_ln=True, out=None):
    """Returns ``(y, mean, rstd)``.  With ``ids`` the input rows are gathered from the table ``x``.
    ``out``: optional preallocated bf16 destination (e.g. a peer-visible all-gather staging buffer)."""
    if use_native(x):
        h = x.shape[-1]
        rows = ids.numel() if ids is not None else x.numel() // h
        y = out if out is not None else torch.empty(rows, h, dtype=torch.bfloat16, device=x.device)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        native().layernorm_fwd(x, ids.reshape(-1) if ids is not None else None, vocab_start, vocab_end,
                               gamma, beta, y, mean, rstd, eps, apply_ln)
        return y, mean, rstd
    if ids is not None:
        flat = ids.reshape(-1)
        mask = (flat >= vocab_start) & (flat < vocab_end)
        src = x[(flat - vocab_start).clamp(0, x.shape[0] - 1)] * mask.unsqueeze(-1).to(x.dtype)
    else:
        src = x.reshape(-1, x.shape[-1])
    if not apply_ln:
        return src, None, None
    xf = src.float()
    mean = xf.mean(-1)
    var = xf.var(-1, unbiased=False)
    rstd = torch.rsqrt(var + eps)
    y = ((xf - mean[:, None]) * rstd[:, None] * gamma.float() + beta.float()).to(src.dtype)
    return y, mean, rstd


def layernorm_bwd(dy, x, gamma, mean, rstd, dx_extra=None, dgamma_acc=None, dbeta_acc=None, dx_out=None):
    """Returns ``(dx, dgamma, dbeta)``; the parameter grads are ``None`` when accumulated in place.  ``dx_out``:
    write dx into this buffer (the next all-gather's staging slot) instead of a fresh tensor."""
    if use_native(dy):
        dx = dx_out if dx_out is not None else torch.empty_like(x)
        if dgamma_acc is None:
            dg = torch.zeros(x.shape[-1], dtype=torch.float32, device=x.device)
            db = torch.zeros_like(dg)
            native().layernorm_bwd(dy, x, gamma, mean, rstd, dx_extra, dx, dg, db)
            return dx, dg.to(gamma.dtype), db.to(gamma.dtype)
        native().layernorm_bwd(dy, x, gamma, mean, rstd, dx_extra, dx, dgamma_acc, dbeta_acc)
        return dx, None, None
    xf, dyf = x.float(), dy.float()
    xhat = (xf - mean[:, None]) * rstd[:, None]
    g = dyf * gamma.float()
    s1 = g.mean(-1, keepdim=True)
    s2 = (g * xhat).mean(-1, keepdim=True)
    dx = rstd[:, None] * (g - s1 - xhat * s2)
    if dx_extra is not None:
        dx = dx + dx_extra.float()
    dgamma = (dyf * xhat).sum(0)
    dbeta = dyf.sum(0)
    if dgamma_acc is not None:
        dgamma_acc.add_(dgamma.to(dgamma_acc.dtype))
        dbeta_acc.add_(dbeta.to(dbeta_acc.dtype))
        return dx.to(x.dtype), None, None
    return dx.to(x.dtype), dgamma.to(gamma.dtype), dbeta.to(gamma.dtype)


def embedding_bwd(dx, ids, vocab_rows, vocab_start, vocab_end, accum_into=None):
    if use_native(dx):
        tgt = accum_into if accum_into is not None else torch.zeros(vocab_rows, dx.shape[-1], dtype=torch.float32, device=dx.device)
        native().embedding_bwd(dx, ids.reshape(-1), tgt, vocab_start, vocab_end, grad_rs_for(accum_into) or {})
        return None if accum_into is not None else tgt.to(dx.dtype)
    flat = ids.reshape(-1)
    mask = (flat >= vocab_start) & (flat < vocab_end)
    g = torch.zeros(vocab_rows, dx.shape[-1], dtype=torch.float32, device=dx.device)
    g.index_add_(0, (flat - vocab_start)[mask], dx.float()[mask])
    if accum_into is not None:
        accum_into.view_as(g).add_(g.to(accum_into.dtype))
        return None
    return g.to(dx.dtype)


# ----------------------------------------------------------------------------------------------
# vocab-parallel cross entropy
# ----------------------------------------------------------------------------------------------
def ce_local_stats(logits, targets, vocab_start):
    """Per row ``(max, sum exp(x - max), target logit or 0)`` over this rank's vocab shard -> [rows, 3] fp32."""
    if use_native(logits):
        stats = torch.empty(logits.shape[0], 3, dtype=torch.float32, device=logits.device)
        native().ce_stats(logits, targets, stats, vocab_start)
        return stats
    lf = logits.float()
    m = lf.max(-1).values
    s = torch.exp(lf - m[:, None]).sum(-1)
    t = targets - vocab_start
    ok = (t >= 0) & (t < logits.shape[1])
    tl = torch.where(ok, lf.gather(1, t.clamp(0, logits.shape[1] - 1)[:, None]).squeeze(1), torch.zeros_like(m))
    return torch.stack([m, s, tl], dim=1)


def ce_partials_buffer(rows: int, vocab_local: int, device) -> torch.Tensor:
    """Buffer for the online-softmax partials the lm_head GEMM epilogue emits: two (max, sumexp) pairs per row and
    256-column tile."""
    return torch.empty(rows, 2 * ((vocab_local + 255) // 256), 2, dtype=torch.float32, device=device)


def ce_stats_from_partials(part, logits, targets, vocab_start):
    """``[rows, 3]`` (max, sum exp(x - max), target logit or 0) from the GEMM epilogue's partials — the statistics pass
    over the ``[rows, vocab]`` logits is gone, only ``rows x tiles x 16`` bytes are read."""
    stats = torch.empty(logits.shape[0], 3, dtype=torch.float32, device=logits.device)
    native().ce_combine(part, logits, targets, stats, vocab_start)
    return stats


def ce_combine_stats(all_stats: torch.Tensor) -> torch.Tensor:
    """Merge ``[T, rows, 3]`` per-shard stats into global ``[rows, 3]`` (max, sumexp, target logit)."""
    m = all_stats[..., 0].max(0).values
    s = (all_stats[..., 1] * torch.exp(all_stats[..., 0] - m)).sum(0)
    tl = all_stats[..., 2].sum(0)
    return torch.stack([m, s, tl], dim=1).contiguous()


def ce_finalize(logits, targets, gstats, vocab_start, grad_scale, ignore_index=-100, write_grad=True):
    """Returns per-row loss; overwrites ``logits`` with ``dlogits * grad_scale`` when ``write_grad``.
    ``grad_scale`` is a 1-element fp32 device tensor (no host sync) or ``None`` (= 1)."""
    if use_native(logits):
        loss_rows = torch.empty(logits.shape[0], dtype=torch.float32, device=logits.device)
        native().ce_finalize(logits, targets, gstats, loss_rows, vocab_start, grad_scale, ignore_index, write_grad)
        return loss_rows
    grad_scale = 1.0 if grad_scale is None else grad_scale.float()
    gm, gs, tl = gstats[:, 0], gstats[:, 1], gstats[:, 2]
    ignored = targets == ignore_index
    loss = torch.where(ignored, torch.zeros_like(gm), torch.log(gs) + gm - tl)
    if write_grad:
        p = torch.exp(logits.float() - gm[:, None]) / gs[:, None]
        t = targets - vocab_start
        ok = (t >= 0) & (t < logits.shape[1]) & ~ignored
        rows = torch.nonzero(ok).squeeze(1)
        p[rows, t[rows]] -= 1.0
        p = p * grad_scale
        p[ignored] = 0
        logits.copy_(p.to(logits.dtype))
    return loss


# ----------------------------------------------------------------------------------------------
# ALiBi causal attention (reference math; the wgmma kernel lives in ops/attention.py)
# ----------------------------------------------------------------------------------------------
def alibi_slopes(n_head: int, device=None) -> torch.Tensor:
    """Per-head ALiBi slopes exactly as transformers' ``build_alibi_tensor`` computes them."""
    closest = 2 ** math.floor(math.log2(n_head))
    base = 2.0 ** (-(2.0 ** -(math.log2(closest) - 3)))
    slopes = torch.pow(torch.tensor(base, dtype=torch.float32), torch.arange(1, 1 + closest, dtype=torch.float32))
    if closest != n_head:
        extra_base = 2.0 ** (-(2.0 ** -(math.log2(2 * closest) - 3)))
        n_rem = min(closest, n_head - closest)
        extra = torch.pow(torch.tensor(extra_base, dtype=torch.float32), torch.arange(1, 1 + 2 * n_rem, 2, dtype=torch.float32))
        slopes = torch.cat([slopes, extra])
    return slopes.to(device)


# ----------------------------------------------------------------------------------------------
# beam search's candidate choice (pipegoose_b200.serving): per request r, whose beams are rows cu_beams[r] ..
# cu_beams[r+1]-1 of logits [N, V], the k best (score, token, row) by score = beam_score[row] + log_softmax(logits[row])
# [token], in fp32, sorted descending; equal scores go to the lower (row, token).
# ----------------------------------------------------------------------------------------------
BEAM_TOPK_MAX_K = 16


def _beam_topk_check(logits: torch.Tensor, cu: list, k: int) -> None:
    V = logits.shape[1]
    if not 1 <= k <= min(BEAM_TOPK_MAX_K, V):
        raise ValueError(f"beam_topk: k must be in 1 .. min({BEAM_TOPK_MAX_K}, V = {V}), got {k}")
    if len(cu) < 2 or cu[0] != 0 or cu[-1] != logits.shape[0] or any(b <= a for a, b in zip(cu, cu[1:])):
        raise ValueError(f"beam_topk: cu_beams must rise from 0 to the {logits.shape[0]} rows, got {cu}")


def beam_topk_reference(logits: torch.Tensor, scores: torch.Tensor, cu_beams, k: int, return_lse: bool = False):
    """fp32 PyTorch form of :func:`beam_topk` (CPU path, test oracle): ``log_softmax``, the add and a stable
    descending sort of each request's flat ``rows * V`` scores."""
    cu = [int(c) for c in cu_beams]
    _beam_topk_check(logits, cu, k)
    x = logits.float()
    lp = torch.log_softmax(x, -1) + scores.to(x.device).float().view(-1, 1)
    V = x.shape[1]
    out_s, out_t, out_r = [], [], []
    for a, b in zip(cu, cu[1:]):
        flat = lp[a:b].reshape(-1)
        idx = torch.sort(flat, descending=True, stable=True).indices[:k]
        out_s.append(flat[idx])
        out_t.append(idx % V)
        out_r.append(idx // V + a)
    out = (torch.stack(out_s), torch.stack(out_t), torch.stack(out_r))
    return out + (torch.logsumexp(x, -1) if return_lse else None,)


def beam_topk(logits: torch.Tensor, scores: torch.Tensor, cu_beams, k: int, return_lse: bool = False):
    """Beam search's candidate choice (section comment above) from ``logits [N, V]`` (bf16 or fp32, rows may be
    strided) and fp32 running scores ``[N]``; ``cu_beams`` is a host sequence of R + 1 ints, at most 64 rows per
    request, and ``k <= 16``.  Returns ``(scores [R, k] fp32, tokens [R, k], rows [R, k], lse [N] or None)``; rows
    index all N rows.  CUDA logits run ``beam_topk_kernel`` (``csrc/beam_sm90.cu``), which reads the logits once."""
    if not logits.is_cuda:
        return beam_topk_reference(logits, scores, cu_beams, k, return_lse)
    from pipegoose_b200.ops.attention import _decode_ticket

    cu = [int(c) for c in cu_beams]
    _beam_topk_check(logits, cu, k)
    if logits.dtype not in (torch.bfloat16, torch.float32) or logits.stride(1) != 1:
        raise ValueError(f"beam_topk: the kernel takes bf16 or fp32 logits with unit inner stride, got {logits.dtype}")
    dev, R = logits.device, len(cu) - 1
    cu_dev = torch.tensor(cu, dtype=torch.int32).to(dev, non_blocking=True)
    out_s = torch.empty(R, k, dtype=torch.float32, device=dev)
    out_t = torch.empty(R, k, dtype=torch.int32, device=dev)
    out_r = torch.empty(R, k, dtype=torch.int32, device=dev)
    lse = torch.empty(logits.shape[0], dtype=torch.float32, device=dev) if return_lse else None
    native().beam_topk(logits, scores.to(dev).float().contiguous(), cu_dev, k, max(b - a for a, b in zip(cu, cu[1:])),
                       out_s, out_t, out_r, lse, _decode_ticket(R, dev))
    return out_s, out_t, out_r, lse
