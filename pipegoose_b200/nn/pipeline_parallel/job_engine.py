"""A pipeline engine built from the job runtime (parity: the reference's execution model, SURVEY §3.5 —
nn/pipeline_parallel/pipeline_engine.py:60-134 + _job/creator.py:182-277): every (micro-batch, partition) task of the
GPipe schedule becomes a ``Job`` created from a ``Package``, jobs are executed by the ``WorkerManager``'s worker
threads, outputs travel as packages, and a ``ProgressTracker`` records which tasks of which clock cycle finished.

What is different from the reference: packages move over PIPELINE-group p2p instead of RPC, the tracker lives in
the c10d store (no sleeps, no per-clock global barriers), and the backward schedule is executed by the engine
instead of being hidden inside an autograd hook of the last micro-batch.  ``PipelineParallel`` installs the static
1F1B engine (pipeline_engine.py) by default; this engine is selected with ``PipelineParallel(..., runtime="jobs")``.
"""
from __future__ import annotations

from queue import Queue
from typing import Dict, List

import torch
from torch import nn

from pipegoose_b200.distributed.parallel_context import ParallelContext
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.nn.pipeline_parallel import microbatch as mb_utils
from pipegoose_b200.nn.pipeline_parallel import queue as Q
from pipegoose_b200.nn.pipeline_parallel._comm import recv_package
from pipegoose_b200.nn.pipeline_parallel._job.creator import create_job, schedule_backward_execution
from pipegoose_b200.nn.pipeline_parallel._job.job import JobStatus
from pipegoose_b200.nn.pipeline_parallel._job.job_type import JobType
from pipegoose_b200.nn.pipeline_parallel._package import Metadata, Package, TrainingMetadata
from pipegoose_b200.nn.pipeline_parallel._utils import get_partition_idx
from pipegoose_b200.nn.pipeline_parallel._worker import WorkerManager
from pipegoose_b200.nn.pipeline_parallel.pipeline_engine import PipelineEngine, _InstallGrads, broadcast_loss_from_last_stage
from pipegoose_b200.nn.pipeline_parallel.scheduler import GPipeScheduler
from pipegoose_b200.nn.pipeline_parallel.sync.handshake import ProgressTracker


class JobPipelineEngine:
    def __init__(self, module: nn.Module, scheduler: GPipeScheduler, parallel_context: ParallelContext,
                 pipeline_context=None, full_module: nn.Module = None, num_workers: int = 1):
        self.module = module  # this rank's stage
        self.full_module = full_module
        self.scheduler = scheduler
        self.parallel_context = parallel_context
        self.pipeline_context = pipeline_context
        self.partition_idx = get_partition_idx(parallel_context)
        self.n_partitions = parallel_context.pipeline_parallel_size
        self.is_first = self.partition_idx == 0
        self.is_last = self.partition_idx == self.n_partitions - 1
        self.tied_group = None
        self.tied_param = None
        # private queues: several engines (tests) may live in one process
        self._pending, self._selected = Queue(), Queue()
        self.worker_manager = WorkerManager(num_workers=num_workers, min_workers=1, max_workers=max(num_workers, 1),
                                            pending_jobs=self._pending, selected_jobs=self._selected)
        self.worker_manager.spawn()
        self.tracker = ProgressTracker(0, parallel_context=parallel_context, parallel_mode=ParallelMode.PIPELINE)
        self._rounds = 0  # how many schedules were published so far (the tracker starts a new round for each)

    # ------------------------------------------------------------------ helpers
    def _run_job(self, job):
        """Hand the job to the worker pool and wait for it (jobs of one stage are ordered by the schedule)."""
        self._pending.put(job)
        assert job.wait(timeout=120), "a pipeline job did not finish"
        if job.status is JobStatus.FAILED or self.worker_manager.failed_jobs:
            err = job.error or self.worker_manager.failed_jobs[-1][1]
            raise RuntimeError(f"pipeline job {job.key} failed") from err
        return job.output

    def _meta(self, i: int, job_type: JobType, src: int, dst: int) -> Metadata:
        return Metadata(i, self.partition_idx, job_type, TrainingMetadata(True, True), src, dst)

    def _init_progress(self, tasks_per_clock: List[List]):
        progress = {c: {(t.microbatch_idx, t.partition_idx): False for t in tasks} for c, tasks in enumerate(tasks_per_clock)}
        if self.parallel_context.get_local_rank(ParallelMode.PIPELINE) == 0:
            self.tracker.initiate(progress)
        # every stage blocks on the store until this round's table is published (no polling, no barrier)
        self.tracker.wait_initiated(self._rounds)
        self._rounds += 1

    # ------------------------------------------------------------------ one training step (GPipe order)
    def run(self, input_ids=None, attention_mask=None, labels=None, **kwargs):
        from pipegoose_b200.models.bloom import CausalLMOutput

        if kwargs.get("position_ids") is not None:
            raise ValueError("PipelineParallel does not take position_ids (packed sequences): micro-batches are cut from "
                             "whole rows without them; train packed batches without pipeline parallelism")
        assert labels is not None, "the job runtime engine implements the training step (pass labels)"
        ctx = self.parallel_context
        me = ctx.get_global_rank()
        prev = ctx.get_prev_global_rank(ParallelMode.PIPELINE)
        nxt = ctx.get_next_global_rank(ParallelMode.PIPELINE)
        inputs = {"input_ids": input_ids, "labels": labels}
        mbs = mb_utils.split({k: v for k, v in inputs.items() if v is not None}, self.scheduler.n_microbatches)
        m = len(mbs)
        weights = PipelineEngine._microbatch_weights(mbs, self.module) if self.is_last else None   # share of the target tokens
        Q.clear_all()
        # the step's gradients are produced from scratch inside this call (see PipelineEngine.train_step): flat fp32
        # main grads are cleared and then held until the optimizer consumed them, ``.grad``s are parked below
        flat = PipelineEngine._flat_state(self)
        if flat is not None:
            flat.hold_grads = False
            flat.zero_grad()
        for p in self.module.parameters():
            p.grad = None
        # data-parallel reducer / tensor-parallel partial-gradient sync: reduce once, after the LAST micro-batch
        reducer = getattr(self.full_module, "_pg_grad_reducer", None) if self.full_module is not None else None
        if reducer is None and self.full_module is not None:
            reducer = getattr(self.full_module, "_pg_tp_grad_sync", None)

        # ---- forward clock cycles
        self._init_progress(self.scheduler.get_forward_schedules())
        outs: Dict[int, Package] = {}
        for i in range(m):
            if self.is_first:
                pkg = Package(mbs[i]["input_ids"], self._meta(i, JobType.FORWARD, me, me))
                fn = (lambda mb: (lambda x: self.module(x)))(mbs[i])
            else:
                pkg = recv_package(prev, ctx)
                if self.is_last:
                    fn = (lambda mb: (lambda x: self.module(x, labels=mb["labels"], batch_seq=tuple(mb["input_ids"].shape))))(mbs[i])
                else:
                    fn = (lambda mb: (lambda x: self.module(x, batch_seq=tuple(mb["input_ids"].shape))))(mbs[i])
            if self.is_first and self.is_last:
                fn = (lambda mb: (lambda x: self.module(x, labels=mb["labels"])))(mbs[i])
            outs[i] = self._run_job(create_job(fn, pkg, ctx, self.pipeline_context))

        # ---- backward clock cycles (reverse micro-batch order, as GPipe)
        self._init_progress(self.scheduler.get_backward_schedules())
        losses = []
        from contextlib import nullcontext

        for n_done, i in enumerate(reversed(range(m)), start=1):
            if self.is_last:
                y = schedule_backward_execution(outs[i]).data   # loss.backward() only records d loss / d output
                loss = y * weights[i]
                losses.append(loss.detach())
                loss.backward()
                grad = Q.get_grad_loss(i, outs[i].metadata.partition_idx)
                pkg = Package(grad, self._meta(i, JobType.BACKWARD, me, me))
            else:
                pkg = recv_package(nxt, ctx)
            with (nullcontext() if (reducer is None or n_done == m) else reducer.no_sync()):
                self._run_job(create_job(self.module, pkg, ctx, self.pipeline_context))
        PipelineEngine.sync_tied_embedding_grad(self)
        if flat is not None:
            flat.hold_grads = True   # survive the zero_grad() that follows forward in the canonical loop
        # the job runtime mirrors the reference: router losses of MoE stages are not part of its objective; drain them so
        # that they (and their graphs) do not pile up across steps
        from pipegoose_b200.nn.expert_parallel.expert_context import ExpertContext

        ExpertContext.get_instance().pop_all_aux_loss(), ExpertContext.get_instance().pop_all_z_loss()
        total = torch.stack(losses).sum() if self.is_last else torch.zeros(())
        total = broadcast_loss_from_last_stage(total, self.parallel_context)
        parked = []
        for p in self.module.parameters():   # re-installed by loss.backward(): a zero_grad() in between cannot lose them
            if p.grad is not None:
                parked.append((p, p.grad))
                p.grad = None
        return CausalLMOutput(loss=_InstallGrads.apply(total.detach().requires_grad_(True), parked, flat), logits=None)

    def destroy(self):
        self.worker_manager.destroy()
