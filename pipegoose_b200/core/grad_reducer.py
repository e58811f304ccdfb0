"""Bucketed, backward-overlapped gradient reduction over the flat fp32 gradient buffer.

Replaces the reference's one blocking ``all_reduce`` per parameter inside an autograd hook
(nn/data_parallel/data_parallel.py:28-43).  The flat gradient buffer is cut into fixed-size
buckets (``BUCKET_SIZE_MB``, constants.py); a bucket is reduced as soon as every parameter in it
has its gradient, on a side stream, while backward keeps running.  Modes:

* ``all_reduce``      every rank ends with the averaged gradients (any optimizer works)
* ``reduce_scatter``  rank ``r`` ends with slice ``r`` of every bucket (what the fused ZeRO-1
                      optimizer consumes) — half the bytes of an all-reduce

On NVLink-connected GPUs the collective is the hand-written peer-memory kernel from
``pipegoose_b200.ops.comm`` (fused with the 1/dp scale); NCCL/gloo is the fallback.
"""
from __future__ import annotations

import os
from contextlib import contextmanager
from typing import Dict, List, Optional

import torch
import torch.distributed as dist
from torch import nn

from pipegoose_b200.constants import BUCKET_SIZE_MB
from pipegoose_b200.core.flat_state import FlatModelState, _ALIGN
from pipegoose_b200.distributed.parallel_mode import ParallelMode


def _tp_all_reduce(t: torch.Tensor, group, comm=None):
    """SUM over the TENSOR group: on the model's NVLink communicator when it offers one, else NCCL / gloo."""
    if comm is not None and getattr(comm, "fused", False):
        comm.all_reduce(t)
    else:
        dist.all_reduce(t, group=group)


def reduce_tp_partial_grads(params, parallel_context, flat: Optional[FlatModelState] = None, comm=None):
    """Sum the gradients of ``tp_partial_grad`` parameters over the TENSOR group, in place.  Gradients live in
    ``param.main_grad`` (flat fp32 buffer: one all-reduce of its head when the tagged parameters are laid out
    there) or, for parameters without a flat state, in ``param.grad`` (gathered into one flat tensor)."""
    if parallel_context.get_world_size(ParallelMode.TENSOR) == 1:
        return
    ps = [p for p in params if getattr(p, "tp_partial_grad", False)]
    if not ps:
        return
    group = parallel_context.get_group(ParallelMode.TENSOR)
    if flat is not None and all(getattr(p, "main_grad", None) is not None for p in ps):
        for p in ps:
            if (p.grad is not None and p.grad.data_ptr() != p.main_grad.data_ptr()
                    and p.grad is not getattr(p, "_pg_materialized", None)):   # (not what materialize_grads exposed)
                # delivered through autograd (e.g. a router's nn.Linear) and not folded yet — without a DataParallel
                # reducer nobody does that before the optimizer step: fold it now so that the sum covers it
                if getattr(p, "_mg_fresh", False):
                    p.main_grad.copy_(p.grad)
                    p._mg_fresh = False
                else:
                    p.main_grad.add_(p.grad)
                p.grad = None
        fresh = [p.main_grad for p in ps if getattr(p, "_mg_fresh", False)]
        if fresh:
            torch._foreach_zero_(fresh)
        for p in ps:
            p._mg_fresh = False
        n = getattr(flat, "tp_partial_numel", 0)
        if all(sum(flat.param_range(p)) <= n for p in ps):
            head = flat.flat_grad[:n]
            # A SUM is not idempotent: a second synced backward in the same gradient window (no zero_grad / optimizer
            # step in between) must only sum its OWN contribution — what the head held after the previous sum is
            # already complete on every rank.
            base = getattr(flat, "tp_reduced_base", None)
            if base is not None and base.numel() == n:
                head.sub_(base)
                _tp_all_reduce(head, group, comm)
                head.add_(base)
            else:
                _tp_all_reduce(head, group, comm)
            flat.tp_reduced_base = head.clone()
            return
    grads = []
    for p in ps:
        g = getattr(p, "main_grad", None)
        if g is None:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            g = p.grad
        elif getattr(p, "_mg_fresh", False):
            g.zero_()
            p._mg_fresh = False
        grads.append(g)
    buf = torch.cat([g.reshape(-1).float() for g in grads])
    dist.all_reduce(buf, group=group)
    torch._foreach_copy_(grads, [f.view_as(g).to(g.dtype) for f, g in zip(buf.split([g.numel() for g in grads]), grads)])


class TensorPartialGradSync:
    """Tensor parallelism WITHOUT a data-parallel reducer (dp == 1): the sequence-parallel layers still produce
    partial gradients for the TP-replicated parameters, so something must sum them over the TENSOR group before
    the optimizer step.  Installed by ``TensorParallel``; steps aside as soon as a :class:`GradReducer` owns the
    module (it does the same reduction in its ``finalize``).  ``no_sync()`` for gradient accumulation: reduce only
    after the last backward of a step."""

    def __init__(self, module: nn.Module, parallel_context):
        self.module = module
        self.ctx = parallel_context
        self._sync = True
        self._queued = False
        self.params = [p for p in module.parameters() if getattr(p, "tp_partial_grad", False)]
        for p in self.params:
            if getattr(p, "_pg_grad_ready", None) is None:
                p._pg_grad_ready = self._on_ready
            if not hasattr(p, "_pg_tp_sync_hook"):
                p._pg_tp_sync_hook = p.register_post_accumulate_grad_hook(self._on_ready)
            if not hasattr(p, "_pg_tp_stash_hook"):
                p._pg_tp_stash_hook = p.register_hook(lambda grad, p=p: self._stash(p, grad))

    def _stash(self, p, grad):
        """Parameters WITHOUT a flat fp32 main grad (a stock ``torch.optim`` on the sequence-parallel model): the partial
        gradient of THIS backward is kept aside instead of being accumulated into ``p.grad``; ``finalize`` sums the
        kept-aside parts over the tensor group and adds the result to ``p.grad``.  A SUM over the group is not idempotent:
        summing ``p.grad`` itself would count an earlier, already complete contribution of the same step T times (two
        backward passes before one optimizer step: gradient accumulation without ``no_sync``, or two losses)."""
        if getattr(p, "main_grad", None) is not None or self._reducer_active():
            return grad
        pending = getattr(p, "_pg_tp_pending", None)
        p._pg_tp_pending = grad.detach().clone() if pending is None else pending.add_(grad)
        return torch.zeros_like(grad)

    def _reducer_active(self) -> bool:
        r = getattr(self.module, "_pg_grad_reducer", None)
        return r is not None and r.flat is not None

    def _on_ready(self, p):
        if self._queued or self._reducer_active():
            return
        self._queued = True
        torch.autograd.Variable._execution_engine.queue_callback(self.finalize)

    def finalize(self):
        self._queued = False
        if not self._sync or self._reducer_active():
            return
        comm = getattr(self.module, "tp", None)
        stashed = [p for p in self.params if getattr(p, "_pg_tp_pending", None) is not None]
        if stashed:
            group = self.ctx.get_group(ParallelMode.TENSOR)
            buf = torch.cat([p._pg_tp_pending.reshape(-1).float() for p in stashed])
            _tp_all_reduce(buf, group, comm)
            for p, part in zip(stashed, buf.split([p.numel() for p in stashed])):
                total = part.view_as(p).to(p.dtype)
                if p.grad is None:
                    p.grad = total.clone()
                else:
                    p.grad.add_(total)
                p._pg_tp_pending = None
        rest = [p for p in self.params if getattr(p, "main_grad", None) is not None]
        if rest:
            reduce_tp_partial_grads(rest, self.ctx, FlatModelState.find(rest), comm=comm)

    @contextmanager
    def no_sync(self):
        prev, self._sync = self._sync, False
        try:
            yield
        finally:
            self._sync = prev


class _Bucket:
    __slots__ = ("index", "start", "end", "params", "pending", "launched", "work", "deferred", "inline")

    def __init__(self, index, start, end):
        self.index, self.start, self.end = index, start, end
        self.params: List[nn.Parameter] = []
        self.pending = 0
        self.launched = False
        self.work = None
        self.deferred = False  # holds TP-partial gradients: reduced over DATA only after the TENSOR all-reduce
        self.inline = False    # reduce-scattered inside the kernels that produce the gradients: never launched here


class GradReducer:
    def __init__(self, module: nn.Module, parallel_context, bucket_size_mb: float = BUCKET_SIZE_MB,
                 mode: str = "all_reduce"):
        self.module = module
        self.ctx = parallel_context
        self.dp = parallel_context.get_world_size(ParallelMode.DATA)
        self.dp_rank = parallel_context.get_local_rank(ParallelMode.DATA)
        self.mode = mode
        self.bucket_size_mb = bucket_size_mb
        self.flat: Optional[FlatModelState] = None
        self.buckets: List[_Bucket] = []
        self._bucket_of: Dict[int, List[_Bucket]] = {}
        self._callback_queued = False
        self._sync = True
        self._fused = None  # set by ops.comm when the NVLink kernels are usable
        self.post_reduce_hooks = []

    # ------------------------------------------------------------------ construction
    def build(self):
        if self.flat is not None:
            return
        gran = self.dp * _ALIGN
        self.bucket_numel = max(gran, int(self.bucket_size_mb * 1024 * 1024 / 4) // gran * gran)
        self.flat = self._make_flat_state()
        # pad the flat buffers so that every bucket (including the last) divides by dp
        n = self.flat.numel
        # With the NVLink engine the small parameters ([0, head): 1-D and tensor-parallel-partial gradients) get a bucket
        # of their own, so that the matrices behind them can leave the bucketed reduction as a whole (enable_inline_rs)
        self.head = self.flat.matrix_start if (self._fused is not None and 0 < self.flat.matrix_start < n) else 0
        self.zero_bucket_numel = self.bucket_numel   # region length the ZeRO-1 slices are cut from (beyond the head)
        self.inline = False
        self.buckets = []
        start, i = 0, 0
        if self.head:
            self.buckets.append(_Bucket(0, 0, self.head))
            start, i = self.head, 1
        while start < n:
            end = min(n, start + self.bucket_numel)
            self.buckets.append(_Bucket(i, start, end))
            start, i = end, i + 1

        def bucket_index(o):
            if self.head:
                return 0 if o < self.head else 1 + (o - self.head) // self.bucket_numel
            return o // self.bucket_numel

        for p in self.flat.params:
            o, cnt = self.flat.param_range(p)
            first, last = bucket_index(o), bucket_index(o + cnt - 1)
            owners = self.buckets[first:last + 1]
            self._bucket_of[id(p)] = owners
            for b in owners:
                b.params.append(p)
                if getattr(p, "tp_partial_grad", False) and self.ctx.get_world_size(ParallelMode.TENSOR) > 1:
                    b.deferred = True
            p._pg_grad_ready = self._on_param_ready
            if not hasattr(p, "_pg_autograd_hook"):
                p._pg_autograd_hook = p.register_post_accumulate_grad_hook(self._on_autograd_grad)
        self._reset_pending()

    def _make_flat_state(self) -> FlatModelState:
        """Flat state in NVLink peer-mapped memory when the fused data-parallel kernels can run
        (CUDA bf16 parameters, NCCL group, dp > 1); plain device memory otherwise."""
        module = self.module
        existing = getattr(module, "_flat_state", None) or FlatModelState.find(module.parameters())
        p0 = next(module.parameters())
        group = self.ctx.get_group(ParallelMode.DATA)
        want_fused = (existing is None and self.dp > 1 and p0.is_cuda and p0.dtype == torch.bfloat16
                      and dist.get_backend(group) == "nccl" and os.environ.get("PIPEGOOSE_B200_FUSED_DP", "1") == "1")
        if want_fused:
            from pipegoose_b200.distributed.symmetric import peers_share_a_node

            want_fused = peers_share_a_node(self.ctx, ParallelMode.DATA)   # replicas on other hosts: NCCL reducer
        if not want_fused:
            return FlatModelState.of(module, pad_to_multiple_of=self.dp)
        from pipegoose_b200.ops.comm import FusedDPEngine

        engine = FusedDPEngine(self.ctx, ParallelMode.DATA)
        state = FlatModelState(module.parameters(), pad_to_multiple_of=self.dp, buffer_factory=engine.allocate)
        module._flat_state = state
        self._fused = engine
        return state

    def enable_inline_rs(self) -> bool:
        """ZeRO-1 with the NVLink engine: the gradients of the matrices ([head, numel), > 99.9 % of the bytes) are
        reduce-scattered by the kernels that produce them — wgrad GEMM epilogue, embedding backward and gradient folds
        ``red.global.add`` every contribution into the owner rank's buffer while backward runs — instead of by bucket
        reductions after them.  Only the small head bucket is still reduced here.  Collective over the DATA group.
        Replaces the reference's per-parameter blocking all-reduce hook (nn/data_parallel/data_parallel.py:28-43)."""
        if self.inline:
            return True
        if self._fused is None or self.mode != "reduce_scatter" or not self.head:
            return False
        if not self._fused.enable_inline(self.head):
            return False
        self.inline = True
        self.flat.inline = self._fused
        self.zero_bucket_numel = self.flat.numel - self.head
        for b in self.buckets:
            b.inline = b.start >= self.head
        for p in self.flat.params:
            if self.flat.param_range(p)[0] >= self.head:
                p._mg_fresh = False     # never overwritten locally: contributions are added at the owners
        self._reset_pending()
        return True

    def _reset_pending(self):
        for b in self.buckets:
            b.pending = sum(getattr(p, "_pg_grad_contribs", 1) for p in b.params)
            b.launched = b.inline
            b.work = None
        self._cursor = len(self.buckets) - 1
        self._contribs_seen: Dict[int, int] = {}

    # ------------------------------------------------------------------ gradient arrival
    def _on_autograd_grad(self, p: nn.Parameter):
        """A gradient delivered through autograd (``p.grad``): fold it into the fp32 main grad."""
        if p.grad is None:
            return
        from pipegoose_b200.ops.functional import acquire_main_grad
        from pipegoose_b200.ops import kernels as K

        mg, accumulate = acquire_main_grad(p, will_overwrite=True)
        K.accumulate_grad(p.grad, mg, accumulate)
        p.grad = None
        self._on_param_ready(p)

    def _on_param_ready(self, p: nn.Parameter):
        if not self._callback_queued:
            self._callback_queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self.finalize)
        if not self._sync or self.dp == 1:
            return
        seen = self._contribs_seen.get(id(p), 0) + 1
        self._contribs_seen[id(p)] = seen
        if seen > getattr(p, "_pg_grad_contribs", 1):
            if any(b.launched and not b.inline for b in self._bucket_of[id(p)]):
                raise RuntimeError(
                    "a gradient contribution arrived after its bucket was reduced: set "
                    "`param._pg_grad_contribs` to the number of contributions per backward pass")
            return
        for b in self._bucket_of[id(p)]:
            b.pending -= 1
        self._launch_ready_in_order()

    def _launch_ready_in_order(self):
        """Reductions are collectives: every replica must issue them in the SAME order.  Buckets are therefore launched
        strictly from the last one down (the order in which a backward pass completes them); a bucket that is ready
        early waits for its predecessors.  A parameter that gets no gradient on THIS replica only (an expert without
        tokens) stalls the cursor here until ``finalize`` launches the rest — in the same descending order — instead of
        letting this replica's sequence of collectives differ from its peers'."""
        i = self._cursor
        while i >= 0:
            b = self.buckets[i]
            if b.deferred or b.launched:
                i -= 1
            elif b.pending == 0:
                self._launch(b)
                i -= 1
            else:
                break
        self._cursor = i

    # ------------------------------------------------------------------ collectives
    def _group_for(self, b: _Bucket):
        return self.ctx.get_group(ParallelMode.DATA)

    def _launch(self, b: _Bucket, tail: bool = False):
        b.launched = True
        for p in b.params:  # parameters that got no gradient this step read as zero
            if getattr(p, "_mg_fresh", False):
                p.main_grad.zero_()
                p._mg_fresh = False
        view = self.flat.flat_grad[b.start:b.end]
        group = self._group_for(b)
        if self._fused is not None:
            if not tail:
                self._fused.begin_overlap()
            b.work = self._fused.reduce_bucket(view, self.mode, tail=tail)
            return
        backend = dist.get_backend(group)
        if backend == "nccl":
            if self.mode == "reduce_scatter":
                n = view.numel() // self.dp
                out = view[self.dp_rank * n:(self.dp_rank + 1) * n]
                b.work = dist.reduce_scatter_tensor(out, view, op=dist.ReduceOp.AVG, group=group, async_op=True)
            else:
                b.work = dist.all_reduce(view, op=dist.ReduceOp.AVG, group=group, async_op=True)
        else:
            view.div_(self.dp)
            b.work = dist.all_reduce(view, op=dist.ReduceOp.SUM, group=group, async_op=True)

    MERGE_TAIL = os.environ.get("PIPEGOOSE_B200_DP_MERGE_TAIL", "0") == "1"

    def _launch_tail(self):
        """Backward is over: reduce what is left.  With the NVLink engine a run of consecutive equally sized buckets (the
        tied embedding table's, which only complete with the last backward kernel: ~45 % of the gradient bytes) goes out
        as ONE launch with one barrier pair instead of one launch per bucket."""
        left = [b for b in reversed(self.buckets) if not b.launched]
        # (merging is opt-in: in a normal backward every bucket has been launched by the time finalize runs — also the tied
        #  table's, which become ready together with the last backward kernel — so this only matters for models that leave
        #  whole runs of buckets without gradients; the multi-bucket form of the kernel is not part of the GPU-validated path)
        if self._fused is None or len(left) < 2 or not self.MERGE_TAIL:
            for b in left:
                self._launch(b, tail=True)
            return
        runs, i = [], 0
        left.sort(key=lambda b: b.index)
        while i < len(left):
            j = i
            uniform = left[i].start >= self.head   # the head bucket has its own length: never merged
            while (uniform and j + 1 < len(left) and left[j + 1].index == left[j].index + 1
                   and left[j].end - left[j].start == self.bucket_numel):
                j += 1
            runs.append(left[i:j + 1])
            i = j + 1
        for run in reversed(runs):
            if len(run) == 1:
                self._launch(run[0], tail=True)
                continue
            for b in run:
                b.launched = True
                for p in b.params:  # parameters that got no gradient this step read as zero
                    if getattr(p, "_mg_fresh", False):
                        p.main_grad.zero_()
                        p._mg_fresh = False
            view = self.flat.flat_grad[run[0].start:run[-1].end]
            run[0].work = self._fused.reduce_bucket(view, self.mode, tail=True, bucket_numel=self.bucket_numel)

    def finalize(self):
        """End of backward: launch what is left, reduce TP-partial gradients, wait for everything."""
        self._callback_queued = False
        if self.flat is None:
            return
        if self._sync:
            self._reduce_tp_partial()  # accumulation steps keep partial sums; only the last backward reduces
        if self._fused is not None:
            self._fused.end_overlap()
        if self._sync and self.dp > 1:
            if self.mode == "reduce_scatter":
                # after a reduce-scatter only slice ``dp_rank`` of a bucket holds reduced values: a second reduction
                # of the same window would average them again.  Accumulate with ``no_sync()`` instead.
                if getattr(self.flat, "reduced_in_window", False):
                    raise RuntimeError(
                        "a second synced backward() reached the ZeRO-1 gradient reduce-scatter before optimizer.step() / "
                        "zero_grad(): wrap every backward of a gradient-accumulation step except the last one in "
                        "`with module.no_sync():`")
            self.flat.reduced_in_window = True
            self._launch_tail()
            for b in self.buckets:
                if b.work is not None:
                    b.work.wait()
            if self.inline:
                # every rank's gradient adds into my slices are complete and visible before the optimizer reads them
                self._fused.barrier()
        else:
            self.flat.finalize_grads()
        if self._sync and not self._fused_optimizer_attached():
            # a stock optimizer (torch.optim.*) reads ``p.grad``: expose the reduced fp32 main grads there
            self.flat.materialize_grads()
        for hook in self.post_reduce_hooks:
            hook()
        self._reset_pending()

    def _fused_optimizer_attached(self) -> bool:
        """FusedAdam (alone or inside DistributedOptimizer) consumes ``main_grad`` directly and marks its parameters."""
        return any(getattr(p, "_pg_fused_optim", False) for p in self.flat.params)

    def _reduce_tp_partial(self):
        """Sequence-parallel layers compute gradients of TP-replicated parameters (LayerNorms,
        row-parallel biases) from their token shard only: sum them over the TENSOR group.  They sit at
        the head of the flat gradient buffer (FlatModelState sorts them first), so this is ONE in-place
        all-reduce; their buckets are held back (``deferred``) until it is enqueued."""
        reduce_tp_partial_grads(self.flat.params, self.ctx, self.flat, comm=getattr(self.module, "tp", None))

    @contextmanager
    def no_sync(self):
        """Skip gradient reduction (gradient accumulation over several backward passes)."""
        prev, self._sync = self._sync, False
        try:
            yield
        finally:
            self._sync = prev
