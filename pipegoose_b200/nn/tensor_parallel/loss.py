"""Vocab-parallel cross entropy (parity: reference nn/tensor_parallel/loss.py:14-103).

Each rank holds ``logits[..., V/T]``.  Only three scalars per token cross the TENSOR group
(row max, sum of exponentials, target logit) — one all-gather of ``[tokens, 3]`` floats instead
of the reference's three all-reduces — and the backward is the true softmax gradient (the
reference saved un-normalised exponentials, Q7).
"""
from __future__ import annotations

import torch
from torch import nn

from pipegoose_b200.distributed.functional import all_gather
from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.nn.tensor_parallel._utils import VocabUtility
from pipegoose_b200.ops import kernels as K


def _kernel_rows(logits2: torch.Tensor, copy: bool = False) -> torch.Tensor:
    """``logits2`` laid out for the cross-entropy kernels, which read rows in 16-byte chunks: a leading dimension that
    is a multiple of 8 elements.  A shard width that is not (GPT-2's 50257 at TP 2 gives 25129 per rank) is copied
    into an 8-padded buffer and handed over as its ``[:, :v_local]`` view; the kernels never read the padding.
    ``copy``: always return a new buffer of that layout (the backward kernel overwrites it in place)."""
    from pipegoose_b200.ops import use_native

    if not copy and (not use_native(logits2) or (logits2.stride(0) % 8 == 0 and logits2.data_ptr() % 16 == 0)):
        return logits2
    rows, v_local = logits2.shape
    buf = torch.empty(rows, (v_local + 7) // 8 * 8, dtype=logits2.dtype, device=logits2.device)
    view = buf[:, :v_local]
    view.copy_(logits2)
    return view


class _VocabParallelCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, parallel_logits: torch.Tensor, targets: torch.Tensor, parallel_context: ParallelContext):
        world = parallel_context.get_world_size(ParallelMode.TENSOR)
        rank = parallel_context.get_local_rank(ParallelMode.TENSOR)
        v_local = parallel_logits.shape[-1]
        vocab_start, _ = VocabUtility.get_vocab_range_idx_from_partition_size(v_local, rank)
        logits2 = parallel_logits.reshape(-1, v_local)
        if not logits2.is_contiguous():
            logits2 = logits2.contiguous()
        logits2 = _kernel_rows(logits2)
        tgt = targets.reshape(-1)
        stats = K.ce_local_stats(logits2, tgt, vocab_start)
        if world > 1:
            gathered = all_gather(stats.unsqueeze(0), dim=0, parallel_context=parallel_context, parallel_mode=ParallelMode.TENSOR)
            gstats = K.ce_combine_stats(gathered)
        else:
            gstats = stats
        loss = torch.log(gstats[:, 1]) + gstats[:, 0] - gstats[:, 2]
        ctx.save_for_backward(logits2, tgt, gstats)
        ctx.vocab_start = vocab_start
        ctx.shape = parallel_logits.shape
        return loss.view(targets.shape).to(torch.float32)

    @staticmethod
    def backward(ctx, grad_output: torch.Tensor):
        logits2, tgt, gstats = ctx.saved_tensors
        from pipegoose_b200.ops import use_native

        g = grad_output.reshape(-1)
        if use_native(logits2) and g.numel() > 0 and (g.stride(0) == 0 or g.numel() == 1):
            # every token carries the same upstream gradient (``loss.mean()`` / ``loss.sum()``): one pass of the fused
            # kernel turns a bf16 copy of the logits into (softmax - onehot) * g — no fp32 [tokens, vocab/T] temporaries
            work = _kernel_rows(logits2, copy=True)
            K.ce_finalize(work, tgt, gstats, ctx.vocab_start, g[:1].float().contiguous(), ignore_index=-(1 << 62), write_grad=True)
            return work.view(ctx.shape), None, None
        p = torch.exp(logits2.float() - gstats[:, 0:1]) / gstats[:, 1:2]
        t = tgt - ctx.vocab_start
        ok = (t >= 0) & (t < logits2.shape[1])
        rows = torch.nonzero(ok).squeeze(1)
        p[rows, t[rows]] -= 1.0
        p = p * grad_output.reshape(-1, 1).float()
        return p.to(logits2.dtype).view(ctx.shape), None, None


class VocabParallelCrossEntropy(nn.Module):
    def __init__(self, parallel_context: ParallelContext):
        super().__init__()
        self.parallel_context = parallel_context

    def forward(self, logits: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        """``logits``: ``[batch, seq, vocab/T]``; ``targets``: ``[batch, seq]``.  Returns the mean token loss."""
        loss = _VocabParallelCrossEntropy.apply(logits, targets, self.parallel_context)
        return loss.mean()
