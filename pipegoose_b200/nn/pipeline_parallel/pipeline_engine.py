"""Pipeline engine: runs this rank's stage through a static schedule with NCCL/gloo point-to-point
transfers between neighbouring stages (parity target: reference
nn/pipeline_parallel/pipeline_engine.py:36-157, which drives the same thing through RPC packages,
worker threads, a progress tracker with per-task sleeps and two global barriers per clock).

Two modes behind ``module.forward``:

* ``model(input_ids, attention_mask)`` (no labels) — **GPipe forward**: returns one output per
  micro-batch (real outputs on the last stage, stand-in scalars elsewhere).  The transfers are
  autograd functions, so the reference's usage ``for out in outputs: out.sum().backward()`` drives
  the backward pipeline on every stage.
* ``model(input_ids, attention_mask, labels=...)`` — **training step**: the engine executes the
  whole schedule (GPipe or 1F1B), backward included, and returns the mean loss.  In the 1F1B steady
  state a stage's send and the receive it waits for next are issued as one batched p2p group, so
  the cross pattern cannot deadlock and transfers overlap with compute.

Activation shapes are static: they are discovered once per micro-batch size by a forward-only
handshake and never sent again (the reference sends dtype/shape/requires_grad with every tensor).
"""
from __future__ import annotations

from contextlib import nullcontext
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import nn

from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.nn.pipeline_parallel import microbatch as mb_utils
from pipegoose_b200.nn.pipeline_parallel._job.job_type import JobType
from pipegoose_b200.nn.pipeline_parallel._utils import get_partition_idx
from pipegoose_b200.nn.pipeline_parallel.scheduler import BaseScheduler
from pipegoose_b200.nn.pipeline_parallel.task import Task



@dataclass
class Schedule:
    """What one rank runs at one clock, in the reference's field order (parity: reference pipeline_engine.py:29-33).
    The schedulers here produce :class:`~pipegoose_b200.nn.pipeline_parallel.task.Task` (hashable, micro-batch first);
    ``Schedule.from_task`` / ``to_task`` convert."""

    job_type: JobType
    partition_idx: int
    microbatch_idx: int

    @classmethod
    def from_task(cls, task: Task) -> "Schedule":
        return cls(task.job_type, task.partition_idx, task.microbatch_idx)

    def to_task(self) -> Task:
        return Task(self.job_type, self.microbatch_idx, self.partition_idx)


def broadcast_loss_from_last_stage(loss: torch.Tensor, parallel_context) -> torch.Tensor:
    """The loss is computed on the last stage; every stage returns it (a 4-byte broadcast over the PIPELINE group,
    enqueued on the stream — no host sync) so that ``loss.item()`` means the same thing on every rank, e.g. for
    logging from global rank 0, which is a first stage."""
    from pipegoose_b200.distributed.parallel_mode import ParallelMode

    if parallel_context.get_world_size(ParallelMode.PIPELINE) == 1:
        return loss
    group = parallel_context.get_group(ParallelMode.PIPELINE)
    src = parallel_context.get_ranks_in_group(ParallelMode.PIPELINE)[-1]
    buf = loss.detach().float().reshape(1).clone()
    if dist.get_backend(group) == "nccl" and not buf.is_cuda:
        buf = buf.cuda()
    dist.broadcast(buf, src=src, group=group)
    return buf.reshape(()).to(loss.device)

class _P2PLink:
    """Point-to-point ops with the previous / next pipeline stage."""

    def __init__(self, ctx: ParallelContext):
        self.ctx = ctx
        self.group = ctx.get_group(ParallelMode.PIPELINE)
        self.is_nccl = dist.get_backend(self.group) == "nccl"
        self.prev = ctx.get_prev_global_rank(ParallelMode.PIPELINE)
        self.next = ctx.get_next_global_rank(ParallelMode.PIPELINE)

    def _device(self):
        return self.ctx.device if self.is_nccl else torch.device("cpu")

    def exchange(self, sends: List[Tuple[torch.Tensor, int]], recvs: List[Tuple[torch.Tensor, int]]):
        """Issue the sends and receives as ONE batched group and wait for completion."""
        ops = [dist.P2POp(dist.isend, t.contiguous(), peer, self.group) for t, peer in sends]
        ops += [dist.P2POp(dist.irecv, t, peer, self.group) for t, peer in recvs]
        if not ops:
            return
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def send_shape(self, shape, dtype, peer):
        from pipegoose_b200.distributed._p2p import DTYPE_TO_ID

        meta = torch.zeros(10, dtype=torch.long)
        meta[0], meta[1] = DTYPE_TO_ID[dtype], len(shape)
        for i, s in enumerate(shape):
            meta[2 + i] = s
        dist.send(meta.to(self._device()), dst=peer, group=self.group)

    def send_object(self, obj, peer):
        """Small Python metadata to a neighbour (handshake only, never in a step)."""
        dist.send_object_list([obj], dst=peer, group=self.group, device=self._device())

    def recv_object(self, peer):
        box = [None]
        dist.recv_object_list(box, src=peer, group=self.group, device=self._device())
        return box[0]

    def recv_shape(self, peer):
        from pipegoose_b200.distributed._p2p import ID_TO_DTYPE

        meta = torch.zeros(10, dtype=torch.long, device=self._device())
        dist.recv(meta, src=peer, group=self.group)
        meta = meta.cpu().tolist()
        return tuple(meta[2:2 + meta[1]]), ID_TO_DTYPE[meta[0]]


class _InstallGrads(torch.autograd.Function):
    """Identity on the loss; backward adds the gradients the pipeline schedule already computed to ``.grad``."""

    @staticmethod
    def forward(ctx, loss, parked, flat=None, engine=None):
        ctx.parked = parked
        ctx.flat = flat
        ctx.engine = engine
        return loss.clone()

    @staticmethod
    def backward(ctx, grad):
        for p, g in ctx.parked:
            p.grad = g if p.grad is None else p.grad + g
        ctx.parked = []
        flat, engine = ctx.flat, ctx.engine
        if engine is not None:
            flat = engine._flat_state()     # (a fused optimizer may have built the flat state after the forward)
        if flat is not None:
            # the window in which a ``zero_grad()`` must be ignored (between forward and this backward) is over: from
            # here on the flat fp32 gradients behave like any accumulated gradients — a ``zero_grad()`` drops them
            flat.hold_grads = False
        if engine is not None:
            # whatever was cleared up to here was cleared BEFORE these gradients were installed: only later clears drop them
            engine._versions_after_schedule = engine._grad_epoch(flat)
        ctx.flat = ctx.engine = None
        return None, None, None, None


class _RecvFromPrev(torch.autograd.Function):
    """forward: receive the activation from the previous stage; backward: send its gradient back."""

    @staticmethod
    def forward(ctx, anchor, link, shape, dtype, device):
        buf = torch.empty(shape, dtype=dtype, device=device)
        link.exchange([], [(buf, link.prev)])
        ctx.link = link
        return buf

    @staticmethod
    def backward(ctx, grad):
        ctx.link.exchange([(grad, ctx.link.prev)], [])
        return None, None, None, None, None


class _SendToNext(torch.autograd.Function):
    """forward: send the activation to the next stage and return a scalar stand-in; backward:
    receive the activation's gradient from the next stage."""

    @staticmethod
    def forward(ctx, act, link):
        link.exchange([(act.detach(), link.next)], [])
        ctx.link = link
        ctx.meta = (act.shape, act.dtype, act.device)
        return act.new_zeros(())

    @staticmethod
    def backward(ctx, _grad_of_standin):
        shape, dtype, device = ctx.meta
        g = torch.empty(shape, dtype=dtype, device=device)
        ctx.link.exchange([], [(g, ctx.link.next)])
        return g, None


class PipelineEngine:
    MASTER_RANK = 0   # the stage that owns the clock in the reference (pipeline_engine.py:39); also the first stage here

    def __init__(self, module: nn.Module, scheduler: BaseScheduler, worker_manager=None,
                 parallel_context: ParallelContext = None, pipeline_context=None, full_module: Optional[nn.Module] = None):
        # ``worker_manager``: the reference's third argument (pipeline_engine.py:36-58); the static runtime executes its
        # schedule on the calling thread and only keeps the object for callers that pass one
        self.worker_manager = worker_manager
        self.module = module  # this rank's stage
        self.full_module = full_module
        self.scheduler = scheduler
        self.parallel_context = parallel_context
        self.pipeline_context = pipeline_context
        self.partition_idx = get_partition_idx(parallel_context)
        self.n_partitions = parallel_context.pipeline_parallel_size
        self.is_first = self.partition_idx == 0
        self.is_last = self.partition_idx == self.n_partitions - 1
        self.link = _P2PLink(parallel_context)
        self._in_meta: Dict[tuple, Tuple[tuple, torch.dtype]] = {}
        self._anchor = None
        self.tied_group = None
        self.tied_param = None
        # weights of the MoE router losses every stage adds to its backward (ExpertLoss defaults; 0 disables a term)
        self.aux_loss_weight = 0.01
        self.z_loss_weight = 0.001

    # ------------------------------------------------------------------ helpers
    def _device(self):
        p = next(self.module.parameters(), None)
        return p.device if p is not None else torch.device("cpu")

    def _stage_accepts(self, name: str) -> bool:
        """Does this stage's ``forward`` take the keyword ``name``?  (Read once from its signature: stage modules are
        plain ``nn.Module``s — the built-in Bloom / GPT-2 / LLaMA-style stages, ``SequentialStage``, or whatever a
        ``UniformPartitioner.register_family`` stage class defines.)"""
        declared = getattr(self.module, "stage_inputs", None)
        if declared is not None:     # a graph stage lists what it reads
            return name in declared
        sig = getattr(self, "_stage_signature", None)
        if sig is None:
            import inspect

            try:
                params = inspect.signature(self.module.forward).parameters
                names = {n for n, p in params.items() if p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)}
                var_kw = any(p.kind is p.VAR_KEYWORD for p in params.values())
            except (TypeError, ValueError):
                names, var_kw = set(), False
            sig = self._stage_signature = (names, var_kw)
        return name in sig[0] or sig[1]

    def _stage_forward(self, x, mb: Dict, with_labels: bool):
        kwargs = {}
        if self._stage_accepts("attention_mask") and mb.get("attention_mask") is not None:
            kwargs["attention_mask"] = mb["attention_mask"]
        if with_labels and self.is_last and self._stage_accepts("labels"):
            kwargs["labels"] = mb["labels"]
        if self._stage_accepts("batch_seq") and "input_ids" in mb:
            kwargs["batch_seq"] = tuple(mb["input_ids"].shape[:2])
        # graph stages (fx_partitioner.GraphStage) name the forward arguments of the traced model they read: every stage
        # holds the micro-batch, so these never travel between stages
        if getattr(self.module, "multi_in", False):
            self.module.select_boundary(self._mb_key(mb))     # which micro-batch shape's metadata unpacks ``x``
        for name in getattr(self.module, "stage_inputs", ()):
            if name in kwargs or (name == "labels" and not (with_labels and self.is_last)):
                continue
            if name in mb:
                kwargs[name] = mb[name]
            elif name == getattr(self.module, "first_input_name", None):
                kwargs[name] = self._first_input(mb)
        return self.module(x, **kwargs)

    def _first_input(self, mb: Dict):
        return mb["input_ids"] if "input_ids" in mb else next(iter(mb.values()))

    def _mb_key(self, mb: Dict) -> tuple:
        return tuple(self._first_input(mb).shape)

    def _handshake(self, microbatches: List[Dict]):
        """Discover this stage's input shape for every distinct micro-batch size (forward-only dry run)."""
        dev = self._device()
        for mb in microbatches:
            key = self._mb_key(mb)
            if key in self._in_meta:
                continue
            with torch.no_grad():
                if self.is_first:
                    x = self._first_input(mb).to(dev)
                    self._in_meta[key] = (tuple(x.shape), x.dtype)
                else:
                    shape, dtype = self.link.recv_shape(self.link.prev)
                    self._in_meta[key] = (shape, dtype)
                    x = torch.zeros(shape, dtype=dtype, device=dev)
                    if getattr(self.module, "multi_in", False):
                        # a graph stage that receives several activations packed into one buffer: their shapes / dtypes
                        self.module.set_in_meta(key, self.link.recv_object(self.link.prev))
                if not self.is_last:
                    out = self._stage_forward(x, {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in mb.items()}, False)
                    self.link.send_shape(tuple(out.shape), out.dtype, self.link.next)
                    if getattr(self.module, "multi_out", False):
                        self.link.send_object(self.module.last_out_meta, self.link.next)

    def _prepare(self, inputs: Dict) -> List[Dict]:
        n = self.scheduler.n_microbatches
        dev = self._device()
        inputs = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in inputs.items() if v is not None}
        mbs = mb_utils.split(inputs, n)
        self._handshake(mbs)
        return mbs

    # ------------------------------------------------------------------ GPipe forward (autograd-driven backward)
    def forward_only(self, inputs: Dict) -> List[torch.Tensor]:
        mbs = self._prepare(inputs)
        dev = self._device()
        if self._anchor is None or self._anchor.device != dev:
            self._anchor = torch.zeros((), device=dev, requires_grad=True)
        outputs = []
        for mb in mbs:
            if self.is_first:
                x = self._first_input(mb)
            else:
                shape, dtype = self._in_meta[self._mb_key(mb)]
                x = _RecvFromPrev.apply(self._anchor, self.link, shape, dtype, dev)
            out = self._stage_forward(x, mb, False)
            outputs.append(out if self.is_last else _SendToNext.apply(out, self.link))
        return outputs

    @torch.no_grad()
    def eval_loss(self, inputs: Dict) -> torch.Tensor:
        """Mean loss over the batch's target tokens, forward only (``with torch.no_grad(): model(ids, labels=...)``)."""
        mbs = self._prepare(inputs)
        dev = self._device()
        weights = self._microbatch_weights(mbs, self.module) if self.is_last else None
        total = torch.zeros((), device=dev)
        for i, mb in enumerate(mbs):
            if self.is_first:
                x = self._first_input(mb)
            else:
                shape, dtype = self._in_meta[self._mb_key(mb)]
                x = torch.empty(shape, dtype=dtype, device=dev)
                self.link.exchange([], [(x, self.link.prev)])
            out = self._stage_forward(x, mb, True)
            if self.is_last:
                total = total + out.float() * weights[i]
            else:
                self.link.exchange([(out.contiguous(), self.link.next)], [])
        return broadcast_loss_from_last_stage(total, self.parallel_context)

    # ------------------------------------------------------------------ scheduled training step
    def _flat_state(self):
        for p in self.module.parameters():
            st = getattr(p, "_pg_flat_state", None)
            if st is not None:
                return st
        return None

    def _grad_epoch(self, flat):
        """Changes whenever the gradients of a schedule were consumed or dropped: FusedAdam counts its steps, a stock
        optimizer updates the parameters in place (their version counters move), a ``zero_grad()`` that really cleared
        the flat fp32 gradients is counted by the flat state."""
        from pipegoose_b200.optim.fused_adam import FusedAdam

        return (sum(p._version for p in self.module.parameters()), FusedAdam.steps_taken, getattr(flat, "clears", 0))

    def _optimizer_stepped_since_last_schedule(self, flat) -> bool:
        """Does this schedule start from scratch (True) or add to the gradients of the previous one (gradient
        accumulation: nothing consumed or dropped them in between)?"""
        last = getattr(self, "_versions_after_schedule", None)
        return last is None or self._grad_epoch(flat) != last

    def train_step(self, inputs: Dict, loss_scale: float = 1.0) -> torch.Tensor:
        # Backward runs inside this call, i.e. BEFORE the user's `optim.zero_grad()` of the canonical loop
        # (`out = model(...); optim.zero_grad(); out.loss.backward(); optim.step()`).  Flat fp32 main grads are
        # cleared here and then held until the optimizer consumed them; autograd `.grad`s are parked and
        # installed by `loss.backward()` (see _InstallGrads).
        # Gradient accumulation: when NO optimizer step happened since the previous schedule, this schedule adds to
        # the gradients that are already there (``loss_scale`` = 1 / number of accumulation steps scales its share).
        flat = self._flat_state()
        fresh = self._optimizer_stepped_since_last_schedule(flat)
        tied_stash = None
        if fresh:
            if flat is not None:
                flat.hold_grads = False
                flat.zero_grad()
            # the schedule produces this step's gradients from scratch: a ``.grad`` left over from the previous step
            # (stock optimizers do not clear it, and zero_grad() only comes after forward) must not be accumulated into
            for p in self.module.parameters():
                p.grad = None
        elif self.tied_group is not None and self.tied_param is not None and (self.is_first or self.is_last):
            # the tied table's gradient is SUMMED over the first and last stage after every schedule: only this
            # schedule's contribution may take part, what is already there was summed before
            g = getattr(self.tied_param, "main_grad", None)
            g = g if g is not None else self.tied_param.grad
            if g is not None:
                tied_stash = g.clone()
                g.zero_()
        mbs = self._prepare(inputs)
        dev = self._device()
        m = len(mbs)
        weights = self._microbatch_weights(mbs, self.module) if self.is_last else None
        if weights is not None and loss_scale != 1.0:
            weights = [w * loss_scale for w in weights]
        order: List[Task] = self.scheduler.get_stage_order(self.partition_idx)
        saved_in: Dict[int, torch.Tensor] = {}
        saved_out: Dict[int, torch.Tensor] = {}
        recv_act: Dict[int, torch.Tensor] = {}
        recv_grad: Dict[int, torch.Tensor] = {}
        saved_aux: Dict[int, torch.Tensor] = {}
        losses = []
        reducer = getattr(self.full_module, "_pg_grad_reducer", None) if self.full_module is not None else None
        if reducer is None and self.full_module is not None:
            reducer = getattr(self.full_module, "_pg_tp_grad_sync", None)  # tp > 1 without data parallelism
        n_bwd_done = 0

        def act_buffer(i):
            shape, dtype = self._in_meta[self._mb_key(mbs[i])]
            return torch.empty(shape, dtype=dtype, device=dev)

        def needs_recv(task: Task):
            if task.job_type is JobType.FORWARD:
                return None if self.is_first or task.microbatch_idx in recv_act else ("act", task.microbatch_idx)
            return None if self.is_last or task.microbatch_idx in recv_grad else ("grad", task.microbatch_idx)

        def post_recv(kind, i, sends):
            if kind == "act":
                buf = act_buffer(i)
                recv_act[i] = buf
                self.link.exchange(sends, [(buf, self.link.prev)])
            else:
                buf = torch.empty_like(saved_out[i])
                recv_grad[i] = buf
                self.link.exchange(sends, [(buf, self.link.next)])

        for idx, task in enumerate(order):
            i = task.microbatch_idx
            need = needs_recv(task)
            if need is not None:
                post_recv(need[0], need[1], [])
            pending_send = None
            if task.job_type is JobType.FORWARD:
                if self.is_first:
                    x = self._first_input(mbs[i])
                else:
                    x = recv_act.pop(i).requires_grad_(True)
                out = self._stage_forward(x, mbs[i], True)
                saved_in[i] = x
                extra = self._moe_auxiliary_loss()   # router losses of THIS stage's MoE layers for this micro-batch
                if self.is_last:
                    loss = out * weights[i]
                    if extra is not None:
                        loss = loss + extra * (loss_scale / m)
                    saved_out[i] = loss
                    losses.append((out * weights[i]).detach() / loss_scale)   # reported: the unscaled language-model loss
                else:
                    saved_out[i] = out
                    if extra is not None:
                        saved_aux[i] = extra * (loss_scale / m)
                    pending_send = (out.detach(), self.link.next)
            else:
                out = saved_out.pop(i)
                x = saved_in.pop(i)
                n_bwd_done += 1
                sync = nullcontext() if (reducer is None or n_bwd_done == m) else reducer.no_sync()
                with sync:
                    if self.is_last:
                        torch.autograd.backward(out)
                    else:
                        aux = saved_aux.pop(i, None)
                        if aux is None:
                            torch.autograd.backward(out, recv_grad.pop(i))
                        else:  # second root: this stage's share of the auxiliary objective
                            torch.autograd.backward([out, aux], [recv_grad.pop(i), torch.ones_like(aux)])
                if not self.is_first:
                    pending_send = (x.grad, self.link.prev)
            if pending_send is not None:
                # pair the send with the receive the next task is going to wait for (1F1B steady state)
                nxt = order[idx + 1] if idx + 1 < len(order) else None
                need_next = needs_recv(nxt) if nxt is not None else None
                if need_next is not None:
                    post_recv(need_next[0], need_next[1], [pending_send])
                else:
                    self.link.exchange([pending_send], [])
        self.sync_tied_embedding_grad()
        if tied_stash is not None:
            g = getattr(self.tied_param, "main_grad", None)
            (g if g is not None else self.tied_param.grad).add_(tied_stash)
        if flat is not None:
            flat.hold_grads = True  # survive the zero_grad() that follows forward in the canonical loop (until backward)
        self._versions_after_schedule = self._grad_epoch(flat)
        if self.is_last:
            total = torch.stack(losses).sum()
        else:
            total = torch.zeros((), device=dev)
        return broadcast_loss_from_last_stage(total, self.parallel_context)

    @staticmethod
    def _microbatch_weights(mbs: List[Dict], stage: Optional[nn.Module] = None) -> List:
        """Share of the step's target tokens that each micro-batch holds, so that the sum of the weighted micro-batch
        (mean) losses IS the mean over all target tokens of the batch — exactly what the unpartitioned model computes,
        also when micro-batches differ in size or in the number of ignored (-100) labels.  Counted on the device.
        A stage that scores fewer positions than "every label but the first" (padding masks) says so through
        ``count_targets(labels, attention_mask)``."""
        m = len(mbs)
        labels = [mb.get("labels") for mb in mbs]
        if any(not isinstance(l, torch.Tensor) for l in labels):
            return [1.0 / m] * m
        count = getattr(stage, "count_targets", None)
        if count is not None:
            counts = torch.stack([count(mb["labels"], mb.get("attention_mask")) for mb in mbs]).float()
        else:
            counts = torch.stack([(l[..., 1:] != -100).sum() for l in labels]).float()
        share = counts / counts.sum().clamp(min=1.0)
        return list(share.unbind(0))

    def _moe_auxiliary_loss(self) -> Optional[torch.Tensor]:
        """Drain the expert context after a stage forward: ``aux_weight * sum(load-balancing) + z_weight * sum(router-z)``
        of the MoE layers this stage ran (None without MoE layers).  Every stage back-propagates its own share — the
        reference leaves the terms of all but the last stage unused, and never drains them."""
        from pipegoose_b200.nn.expert_parallel.expert_context import ExpertContext

        store = ExpertContext.get_instance()
        aux, z = store.pop_all_aux_loss(), store.pop_all_z_loss()
        terms = [self.aux_loss_weight * t for t in aux if self.aux_loss_weight] + \
                [self.z_loss_weight * t for t in z if self.z_loss_weight]
        terms = [t for t in terms if isinstance(t, torch.Tensor) and t.requires_grad]
        if not terms:
            return None
        return torch.stack([t.float().reshape(()) for t in terms]).sum()

    def sync_tied_embedding_grad(self):
        """Sum the tied embedding / lm_head table's gradient over the first and last stage."""
        if self.tied_group is None or self.tied_param is None or not (self.is_first or self.is_last):
            return
        p = self.tied_param
        g = getattr(p, "main_grad", None)
        if g is None:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            g = p.grad
        t = g if dist.get_backend(self.tied_group) != "nccl" or g.is_cuda else g.cuda()
        dist.all_reduce(t, group=self.tied_group)
        if t is not g:
            g.copy_(t)
        flat = getattr(p, "_pg_flat_state", None)
        if (flat is not None and getattr(flat, "grads_materialized", False) and p.grad is not None
                and p.grad.data_ptr() != g.data_ptr()):
            # the data-parallel reducer already exposed the (pre-sum) main grad as a ``.grad`` COPY for a stock optimizer
            p.grad = g.to(p.dtype)

    # ------------------------------------------------------------------ entry point used as module.forward
    def run(self, input_ids=None, attention_mask=None, labels=None, **kwargs):
        """``loss_scale`` (keyword): factor on this call's gradients — pass ``1 / k`` on each of the ``k`` calls of a
        gradient-accumulation step (the backward pass runs inside this call, a later ``(loss / k).backward()`` cannot
        scale it any more).  The returned loss is unscaled."""
        if kwargs.get("position_ids") is not None:
            raise ValueError("PipelineParallel does not take position_ids (packed sequences): micro-batches are cut from "
                             "whole rows without them; train packed batches without pipeline parallelism")
        inputs = {"input_ids": input_ids, "attention_mask": attention_mask, "labels": labels}
        inputs.update(kwargs)
        if labels is None:
            return self.forward_only(inputs)
        from pipegoose_b200.models.bloom import CausalLMOutput

        if not torch.is_grad_enabled():   # evaluation: the loss only, no schedule, nothing touches the gradients
            inputs.pop("loss_scale", None)
            return CausalLMOutput(loss=self.eval_loss(inputs), logits=None)

        loss = self.train_step(inputs, loss_scale=float(inputs.pop("loss_scale", 1.0) or 1.0))
        # backward already ran inside the schedule.  Gradients that live in `.grad` are parked and re-installed
        # by `loss.backward()`, so a `zero_grad()` between forward and backward does not lose them.
        parked = []
        for p in self.module.parameters():
            if p.grad is not None:  # autograd grads, or main grads the data-parallel reducer materialised
                parked.append((p, p.grad))
                p.grad = None
        return CausalLMOutput(loss=_InstallGrads.apply(loss.detach().requires_grad_(True), parked, None, self), logits=None)
