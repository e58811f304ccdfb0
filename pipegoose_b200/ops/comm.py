"""Fused compute+collective engines over NVLink peer memory.

``FusedTPEngine`` drives the two tensor-parallel kernels

* **all-gather -> GEMM** (`ag_gemm`, `ag_gemm_nn`): ONE launch of the wgmma GEMM kernel in which
  a few communication CTAs pull every peer's activation shard through NVSwitch with bulk async
  copies into the local gathered operand while the remaining CTAs run the MMA tiles, visiting the
  row chunks in arrival order (local shard first) and acquiring a per-chunk counter before the
  TMA loads of that chunk;
* **GEMM -> reduce-scatter** (`gemm_rs`, `gemm_rs_nn`): the GEMM epilogue stores each output tile
  straight into the owner rank's staging slot (peer ``st.global``) and bumps the owner's arrival
  counter; a small reduce kernel on the owner sums the T partial tiles with bias and residual as
  soon as the counters say they landed.

Buffers are double-buffered by operation parity; all flags/counters are monotonic (no resets).
"""
from __future__ import annotations

from typing import Optional

import torch

from pipegoose_b200.distributed import symmetric as S
from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops import native

_BM = 128
import os

N_COMM_CTAS = int(os.environ.get("PIPEGOOSE_B200_NCOMM", "16"))
# 1: GEMM -> reduce-scatter reduces the local chunk in its own epilogue (no reduce kernel, but the staged partials are
# read without prefetch); 0 (default): separate rs_reduce kernel
RS_FUSED_REDUCE = os.environ.get("PIPEGOOSE_B200_RS_FUSED_REDUCE", "0") == "1"


def pick_tiling(rows: int, n: int, k: int, chunks: int, ctas: int) -> int:
    """``block_n`` for a GEMM -> reduce-scatter: mirror of ``pick_bn`` in csrc/gemm_sm90.cu (the arrival counters of a
    reduce-scatter are counted in tiles, so both sides must agree on the tiling)."""
    best, best_cost = 256, float("inf")
    for bn, eff in ((256, 1.0), (192, 0.93), (128, 0.82), (64, 0.55)):
        if bn > 64 and n <= bn // 2:
            continue
        tiles = ((rows + _BM - 1) // _BM) * ((n + bn - 1) // bn) * chunks
        waves = (tiles + ctas - 1) // ctas
        cost = waves * bn / eff
        if cost < best_cost * 0.97:
            best, best_cost = bn, cost
    return best


class FusedTPEngine:
    def __init__(self, comm, ag_bytes: int = 0, rs_bytes: int = 0):
        self.comm = comm
        self.T = comm.size
        self.rank = comm.rank
        self.ctx = comm.ctx
        self.mode = comm.mode
        self.ws: Optional[S.SymmetricWorkspace] = None
        self._ag_slot_bytes = 0
        self._rs_slot_bytes = 0
        self.ag_epoch = 0
        self.rs_calls = 0
        self.rs_expected = 0
        self.num_sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        self._dummy = {}

    # ------------------------------------------------------------------ workspace
    def _ensure(self, ag_slot: int, rs_slot: int):
        ag_slot = (ag_slot + 1023) // 1024 * 1024
        rs_slot = (rs_slot + 1023) // 1024 * 1024
        if self.ws is not None and ag_slot <= self._ag_slot_bytes and rs_slot <= self._rs_slot_bytes:
            return
        self._ag_slot_bytes = max(self._ag_slot_bytes, ag_slot)
        self._rs_slot_bytes = max(self._rs_slot_bytes, rs_slot)
        if self.ws is not None:
            self.ws.close()
        total = 2 * self._ag_slot_bytes + 2 * self._rs_slot_bytes
        self.ws = S.SymmetricWorkspace(self.ctx, self.mode, total)
        self.ag_epoch = 0
        self.rs_calls = 0
        self.rs_expected = 0

    def _ag_off(self, slot: int) -> int:
        return slot * self._ag_slot_bytes

    def _rs_off(self, slot: int) -> int:
        return 2 * self._ag_slot_bytes + slot * self._rs_slot_bytes

    def _dummy_out(self, n: int, device):
        t = self._dummy.get(n)
        if t is None:
            t = torch.empty(1, n, dtype=torch.bfloat16, device=device)
            self._dummy[n] = t
        return t

    def supports(self, rows_local: int) -> bool:
        return rows_local % _BM == 0

    # ------------------------------------------------------------------ all-gather -> GEMM
    def ag_input_buffer(self, rows_local: int, cols: int) -> Optional[torch.Tensor]:
        """The peer-visible staging buffer the NEXT all-gather will publish: producers (LayerNorm)
        write their output straight into it so no copy precedes the fused kernel."""
        if not self.supports(rows_local):
            return None
        self._ensure(rows_local * cols * 2, self._rs_slot_bytes)
        slot = (self.ag_epoch + 1) & 1
        return self.ws.local_tensor(self._ag_off(slot), (rows_local, cols), torch.bfloat16)

    def _ag_gemm(self, x_shard, weight, b_mn, bias, flags, aux, out_cols, extra=None):
        T, r = self.T, self.rank
        m_local, k = x_shard.shape
        m = m_local * T
        shard_bytes = m_local * k * 2
        # largest reduce-scatter staging seen so far is kept; grow lazily (collective)
        self._ensure(shard_bytes, self._rs_slot_bytes)
        ws = self.ws
        self.ag_epoch += 1
        slot = self.ag_epoch & 1
        stage = ws.local_tensor(self._ag_off(slot), (m_local, k), torch.bfloat16)
        if x_shard.data_ptr() != stage.data_ptr():
            stage.copy_(x_shard)
        x_full = torch.empty(m, k, dtype=torch.bfloat16, device=x_shard.device)
        out = torch.empty(m, out_cols, dtype=torch.bfloat16, device=x_shard.device)
        ag = dict(
            n_comm=N_COMM_CTAS, dst=x_full.data_ptr(), chunk_bytes=shard_bytes,
            ready=ws.sig_ptr(r, S.SIG_AG_READY), epoch=self.ag_epoch, rank=r, local=stage.data_ptr(),
            src=[ws.data_ptr(p, self._ag_off(slot)) for p in range(T)],
            peer_flag=[ws.sig_ptr(p, S.SIG_AG_READY + r) for p in range(T)],
        )
        if extra:
            ag.update(extra)
        native().gemm(x_full, weight, out, False, b_mn, bias, None, aux, flags, 0, 0,
                      T, r, ws.sig_ptr(r, S.SIG_CHUNK_CTR), N_COMM_CTAS * self.ag_epoch, [], [], ag)
        return out, x_full

    def ag_gemm(self, x_shard, weight, bias=None, gelu=False, aux_holder=None, extra=None):
        """``(gather(x) @ W^T + b [gelu], gather(x))`` with ``x_shard`` = this rank's token shard.  ``extra``: more
        epilogue arguments for the kernel (``ce_part`` / ``ce_valid`` of the lm_head)."""
        if not self.supports(x_shard.shape[0]):
            x_full = self.comm.all_gather_rows(x_shard)
            z = torch.empty(x_full.shape[0], weight.shape[0], dtype=x_full.dtype, device=x_full.device) if gelu else None
            y = K.gemm_nt(x_full, weight, bias, gelu=gelu, aux_out=z, **({"ag": extra} if extra else {}))
            if aux_holder is not None:
                aux_holder["aux"] = z
            return y, x_full
        aux = None
        if gelu:
            aux = torch.empty(x_shard.shape[0] * self.T, weight.shape[0], dtype=torch.bfloat16, device=x_shard.device)
            if aux_holder is not None:
                aux_holder["aux"] = aux
        return self._ag_gemm(x_shard.contiguous(), weight, False, bias, K.EPI_GELU if gelu else 0, aux, weight.shape[0],
                             extra=extra)

    def ag_gemm_nn(self, dy_shard, weight, dgelu_aux=None):
        """``(gather(dy) @ W [* gelu'(aux)], gather(dy))`` — dgrad of a row-parallel linear."""
        if not self.supports(dy_shard.shape[0]):
            dy_full = self.comm.all_gather_rows(dy_shard)
            return K.gemm_nn(dy_full, weight, dgelu_aux=dgelu_aux), dy_full
        flags = K.EPI_DGELU if dgelu_aux is not None else 0
        return self._ag_gemm(dy_shard.contiguous(), weight, True, None, flags, dgelu_aux, weight.shape[1])

    # ------------------------------------------------------------------ GEMM -> reduce-scatter
    def _gemm_rs(self, a, weight, b_mn, bias, residual, n):
        T, r = self.T, self.rank
        m = a.shape[0]
        m_local = m // T
        slot_bytes = T * m_local * n * 2
        self._ensure(self._ag_slot_bytes, slot_bytes)
        ws = self.ws
        self.rs_calls += 1
        slot = self.rs_calls & 1
        k = a.shape[1]
        bn = pick_tiling(m_local, n, k, T, self.num_sms)
        # every CTA bumps the owner's counter once per tile it stored
        tiles_per_chunk = ((m_local + _BM - 1) // _BM) * ((n + bn - 1) // bn)
        self.rs_expected += tiles_per_chunk
        src_stride = m_local * n  # elements between two sources' slots
        out_peer = [ws.data_ptr(p, self._rs_off(slot) + r * src_stride * 2) for p in range(T)]
        arrive = [ws.sig_ptr(p, S.SIG_RS_ARRIVE + r) for p in range(T)]
        out = torch.empty(m_local, n, dtype=torch.bfloat16, device=a.device)
        if RS_FUSED_REDUCE:
            # the epilogue of this rank's own (last visited) chunk adds the peers' staged partials + bias + residual
            ag = {"rank": r, "rs_wait": ws.sig_ptr(r, S.SIG_RS_ARRIVE),
                  "rs_wait_value": self.rs_expected,
                  "rs_in": [ws.data_ptr(r, self._rs_off(slot) + s * src_stride * 2) for s in range(T)]}
            native().gemm(a, weight, out, False, b_mn, bias, residual, None, 0, bn, 0,
                          T, (r + 1) % T, 0, 0, out_peer, arrive, ag)
            return out
        native().gemm(a, weight, self._dummy_out(n, a.device), False, b_mn, None, None, None, 0, bn, 0,
                      T, (r + 1) % T, 0, 0, out_peer, arrive, {})
        native().rs_reduce(ws.data_ptr(r, self._rs_off(slot)), T, src_stride, ws.sig_ptr(r, S.SIG_RS_ARRIVE),
                           self.rs_expected, bias, residual, out)
        return out

    def gemm_rs(self, a, weight, bias=None, residual=None):
        """``reduce_scatter_rows(a @ W^T) + b + residual`` — forward of a row-parallel linear."""
        if not self.supports(a.shape[0] // self.T):
            y = self.comm.reduce_scatter_rows(K.gemm_nt(a, weight))
            if bias is not None:
                y = y + bias
            return y + residual if residual is not None else y
        return self._gemm_rs(a.contiguous(), weight, False, bias, residual, weight.shape[0])

    def gemm_rs_nn(self, dy, weight):
        """``reduce_scatter_rows(dy @ W)`` — dgrad of a column-parallel linear."""
        if not self.supports(dy.shape[0] // self.T):
            return self.comm.reduce_scatter_rows(K.gemm_nn(dy, weight))
        return self._gemm_rs(dy.contiguous(), weight, True, None, None, weight.shape[1])


    # ------------------------------------------------------------------ small collectives on peer memory
    # The vocab-parallel embedding (reduce-scatter forward, all-gather backward), the cross-entropy statistics exchange
    # and the tensor-group sum of the sequence-parallel partial gradients: no GEMM to fuse them into, but they run on
    # the same NVLink protocols instead of NCCL, so a tensor-parallel step contains no library collective.
    PUSH_BLOCKS = 32

    def reduce_scatter_rows(self, x: torch.Tensor) -> torch.Tensor:
        """``[T * rows, n]`` partial sums -> this rank's ``[rows, n]`` block of the sum: row block c is pushed into
        rank c's staging slot (the GEMM -> reduce-scatter protocol without a GEMM), the owner sums the T slots."""
        T, r = self.T, self.rank
        x = x.contiguous()
        m, n = x.shape
        m_local = m // T
        self._ensure(self._ag_slot_bytes, T * m_local * n * 2)
        ws = self.ws
        self.rs_calls += 1
        slot = self.rs_calls & 1
        self.rs_expected += self.PUSH_BLOCKS
        src_stride = m_local * n
        out_peer = [ws.data_ptr(p, self._rs_off(slot) + r * src_stride * 2) for p in range(T)]
        arrive = [ws.sig_ptr(p, S.SIG_RS_ARRIVE + r) for p in range(T)]
        native().rs_push(x, T, (r + 1) % T, out_peer, arrive, self.PUSH_BLOCKS)
        out = torch.empty(m_local, n, dtype=torch.bfloat16, device=x.device)
        native().rs_reduce(ws.data_ptr(r, self._rs_off(slot)), T, src_stride, ws.sig_ptr(r, S.SIG_RS_ARRIVE),
                           self.rs_expected, None, None, out)
        return out

    def _misc(self, nbytes: int) -> S.SymmetricWorkspace:
        """A second, small workspace (own flags) for the all-gather / all-reduce kernels below; grown collectively."""
        nbytes = (nbytes + 4095) // 4096 * 4096
        ws = getattr(self, "_misc_ws", None)
        if ws is None or ws.nbytes < 2 * nbytes:
            if ws is not None:
                ws.close()
            self._misc_ws = ws = S.SymmetricWorkspace(self.ctx, self.mode, 2 * nbytes)
            self._misc_slot_bytes = nbytes
            self._misc_epoch = 0
            self._misc_calls = 0
        return ws

    def all_gather_rows(self, x_shard: torch.Tensor) -> torch.Tensor:
        """``[rows, ...]`` -> ``[T * rows, ...]`` (any 2-byte or 4-byte dtype): every rank places its shard in its own
        copy of the gathered buffer and pushes it to all peers in one kernel that ends with a peer barrier."""
        T, r = self.T, self.rank
        x_shard = x_shard.contiguous()
        shard_bytes = x_shard.numel() * x_shard.element_size()
        assert shard_bytes % 16 == 0
        ws = self._misc(T * shard_bytes)
        self._misc_calls += 1
        off = (self._misc_calls & 1) * self._misc_slot_bytes
        full = ws.local_tensor(off, (T * x_shard.shape[0],) + tuple(x_shard.shape[1:]), x_shard.dtype)
        full[r * x_shard.shape[0]:(r + 1) * x_shard.shape[0]].copy_(x_shard)
        self._misc_epoch += 1
        total = T * shard_bytes // 2   # in bf16 elements
        native().allgather_bf16([ws.data_ptr(p, off) for p in range(T)], r, total, total,
                                [ws.sig_ptr(p, S.SIG_BARRIER) for p in range(T)], self._misc_epoch, 0, 0)
        return full

    def all_reduce_f32_(self, t: torch.Tensor) -> torch.Tensor:
        """In-place SUM of a small contiguous fp32 tensor over the group (two-shot kernel on peer memory)."""
        T, r = self.T, self.rank
        n = t.numel()
        pad = (n + T * 4 - 1) // (T * 4) * (T * 4)
        ws = self._misc(pad * 4)
        self._misc_calls += 1
        off = (self._misc_calls & 1) * self._misc_slot_bytes
        buf = ws.local_tensor(off, (pad,), torch.float32)
        buf[:n].copy_(t.reshape(-1))
        if pad > n:
            buf[n:].zero_()
        self._misc_epoch += 1
        native().allreduce_f32([ws.data_ptr(p, off) for p in range(T)], r, 0, pad, 1.0, False,
                               [ws.sig_ptr(p, S.SIG_BARRIER) for p in range(T)], self._misc_epoch, 8, 0)
        t.reshape(-1).copy_(buf[:n])
        return t


class _StreamWork:
    """`Work`-like handle: the collective ran on a side stream; ``wait`` orders the caller's stream after it."""

    def __init__(self, event):
        self.event = event

    def wait(self):
        torch.cuda.current_stream().wait_event(self.event)


class FusedDPEngine:
    """Data-parallel gradient reduction and ZeRO-1 parameter all-gather as hand-written NVLink kernels.

    The flat fp32 gradient buffer and the flat bf16 parameter buffer live in a peer-mapped workspace.
    ``reduce_bucket`` launches (on a side stream, overlapped with backward) a two-shot kernel: every
    rank pulls slice ``r`` of the bucket from all peers, sums it, scales by 1/dp and - for
    all-reduce - pushes the result to all peers; for ZeRO-1 (reduce-scatter) it keeps the slice.
    ``all_gather_params`` pushes this rank's updated bf16 slices of every bucket to all peers in
    one launch.
    """

    def __init__(self, parallel_context, parallel_mode):
        self.ctx = parallel_context
        self.mode = parallel_mode
        self.world = parallel_context.get_world_size(parallel_mode)
        self.rank = parallel_context.get_local_rank(parallel_mode)
        self.ws: Optional[S.SymmetricWorkspace] = None
        self.epoch = 0
        self.stream = torch.cuda.Stream()
        self._grad_off = 0
        self._param_off = 0

    def allocate(self, numel: int, param_dtype, grad_dtype):
        assert param_dtype == torch.bfloat16 and grad_dtype == torch.float32
        grad_bytes = numel * 4
        param_bytes = numel * 2
        self._grad_off = 0
        self._param_off = (grad_bytes + 1023) // 1024 * 1024
        self.ws = S.SymmetricWorkspace(self.ctx, self.mode, self._param_off + param_bytes)
        grad = self.ws.local_tensor(self._grad_off, (numel,), torch.float32)
        param = self.ws.local_tensor(self._param_off, (numel,), torch.bfloat16)
        self._grad_base = grad.data_ptr()
        self._grad = grad
        self.numel = numel
        self.inline_start = None     # first element of the in-kernel reduce-scatter region (None: off)
        self.inline_dirty = False    # a kernel added gradients into the region since the owners last cleared it
        # NVLS (multicast object bound to the workspace): reduce with multimem.ld_reduce, all-gather with multimem.st
        def want(mode):
            return mode == "1" or (mode == "auto" and self.world >= 4)

        self._mc_grad = self.ws.mc_data_ptr(self._grad_off) if want(self.NVLS_REDUCE) else 0
        self._mc_param = self.ws.mc_data_ptr(self._param_off) if want(self.NVLS_ALLGATHER) else 0
        return param, grad

    # NVLS (multimem.ld_reduce / multimem.st through the NVSwitch multicast object): "auto" = groups of >= 4 ranks.
    # With ONE peer the switch-side reduction saves no bytes and adds latency; from 4 ranks on a pull through the switch
    # moves 1/world of the bytes of a pull from every peer.
    NVLS_REDUCE = os.environ.get("PIPEGOOSE_B200_NVLS_REDUCE", "auto")
    NVLS_ALLGATHER = os.environ.get("PIPEGOOSE_B200_NVLS_ALLGATHER", "auto")
    # 1: reduce-scatter the matrices' gradients inside the kernels that produce them (red.global.add into the owner's
    # buffer).  OFF by default: NVLink remote atomics run far below the bandwidth of plain peer loads / stores and the
    # wgrad epilogues stall on them (the earlier sm_100a build measured it slower than the bucketed reducer; not
    # re-measured on H100).  Kept as an option and as a tested kernel path.
    INLINE_RS = os.environ.get("PIPEGOOSE_B200_DP_INLINE_RS", "0") == "1"
    # 1: four scalar red.global.add.f32 per 16 bytes instead of one red.global.add.v4.f32 (diagnosis)
    INLINE_SCALAR_RED = os.environ.get("PIPEGOOSE_B200_DP_INLINE_SCALAR", "0") == "1"

    # ------------------------------------------------------------------ in-kernel gradient reduce-scatter (ZeRO-1)
    def enable_inline(self, start: int) -> bool:
        """Gradients of flat elements [start, numel) are from now on added by the kernels that produce them (wgrad GEMM
        epilogue, embedding backward, gradient folds) straight into the buffer of the rank owning their ZeRO-1 slice
        (``red.global.add`` over NVLink): no bucket reduction, nothing exposed after backward but one peer barrier."""
        if not self.INLINE_RS or self.world < 2 or start >= self.numel:
            return False
        n = self.numel - start
        assert n % (self.world * 4) == 0 and start % 4 == 0
        self.inline_start = start
        self.inline_seg = n // self.world
        desc = {"peer": [self.ws.data_ptr(p, self._grad_off) for p in range(self.world)],
                "local": self.ws.data_ptr(self.rank, self._grad_off), "start": start, "seg": self.inline_seg,
                "scalar": 1 if self.INLINE_SCALAR_RED else 0}
        K.register_grad_rs(self._grad_base + start * 4, self._grad_base + self.numel * 4, desc, self)
        self._grad[start:].zero_()
        self.barrier()
        return True

    def barrier(self):
        """Peer barrier on the current stream: what every rank of the group enqueued before it (gradient adds into my
        buffer included) is complete and visible to what I enqueue after it."""
        self.epoch += 1
        native().barrier_peers(self._flag_ptrs(), self.rank, self.epoch)

    def clear_inline_region(self, force: bool = False):
        """``zero_grad`` of the in-kernel region when its gradients were produced but not consumed by an optimizer step
        (the step clears the owner slices while it reads them).  Collective: peers may not add before everyone cleared."""
        if self.inline_start is None or not (self.inline_dirty or force):
            return
        self.barrier()                      # nobody is still adding into my buffer ...
        self._grad[self.inline_start:].zero_()
        self.barrier()                      # ... and nobody starts before every buffer is clear
        self.inline_dirty = False

    def inline_consumed(self):
        self.inline_dirty = False

    def close_inline(self):
        K.unregister_grad_rs(self)
        self.inline_start = None

    def __del__(self):   # a dead engine's address range must not capture gradients of later allocations
        try:
            K.unregister_grad_rs(self)
        except Exception:
            pass

    def _flag_ptrs(self):
        return [self.ws.sig_ptr(p, S.SIG_BARRIER) for p in range(self.world)]

    # CTAs of a gradient reduction that overlaps backward / runs after it.  Positive: 512-thread CTAs; negative: that many
    # CTAs of the small form (128 threads, <= 64 registers, see csrc/comm.cu).  A persistent GEMM CTA holds its SM's whole
    # register file, so while reductions overlap backward the GEMM grids are capped to leave |OVERLAP_CTAS| SMs to the
    # reducer (CAP_GEMMS): a reducer CTA, which waits on peers inside the kernel, then never keeps a GEMM CTA from
    # becoming resident.  The tail reductions run after the last backward kernel, and finalize() orders the compute
    # stream after them, so no GEMM runs next to them.  16 CTAs keep ~1 MB in flight over NVLink (8 x 16 B loads per
    # thread), about the bandwidth-delay product of one NVLink4 direction; the tail uses 48 (one per ~3 SMs of 132).
    OVERLAP_CTAS = int(os.environ.get("PIPEGOOSE_B200_DP_OVERLAP_CTAS", "16"))
    TAIL_CTAS = int(os.environ.get("PIPEGOOSE_B200_DP_TAIL_CTAS", "48"))
    # 0: GEMM grids keep every SM while reductions overlap backward; the reducer then depends on GEMM kernel boundaries
    # to become resident, and a tensor-parallel GEMM that waits on a peer can stall it — only for experiments
    CAP_GEMMS = os.environ.get("PIPEGOOSE_B200_DP_CAP_GEMMS", "1") == "1"

    def begin_overlap(self):
        """Backward starts reducing buckets: persistent GEMM grids leave ``|OVERLAP_CTAS|`` SMs to the reducer (a
        reducer CTA occupies at most one SM; a persistent GEMM whose CTAs cannot all be resident stalls behind it)."""
        if self.CAP_GEMMS and not getattr(self, "_capped", False):
            sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
            native().set_gemm_cta_cap(max(1, sms - abs(self.OVERLAP_CTAS)))
            self._capped = True

    def end_overlap(self):
        if getattr(self, "_capped", False):
            native().set_gemm_cta_cap(0)
            self._capped = False

    def reduce_bucket(self, view: torch.Tensor, mode: str, tail: bool = False, bucket_numel: int = 0):
        """``view``: one bucket, or (``bucket_numel`` > 0) a run of consecutive buckets of that size reduced by ONE
        launch — each bucket slice-wise, so that ZeRO-1 ownership does not depend on how launches were merged."""
        offset = (view.data_ptr() - self._grad_base) // 4
        n = view.numel()
        ready = torch.cuda.Event()
        ready.record()  # gradients of this bucket were produced on the current stream
        self.epoch += 1
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            native().allreduce_f32([self.ws.data_ptr(p, self._grad_off) for p in range(self.world)], self.rank,
                                   offset, n, 1.0 / self.world, mode == "reduce_scatter", self._flag_ptrs(), self.epoch,
                                   self.TAIL_CTAS if tail else self.OVERLAP_CTAS, self._mc_grad, bucket_numel)
            done = torch.cuda.Event()
            done.record()
        return _StreamWork(done)

    def all_gather_params(self, flat_param: torch.Tensor, bucket_numel: int, head: int = 0):
        """Regions [0, head) and [head + k * bucket_numel, ...): every rank pushes its 1/world slice of each region to all
        peers — with NVLS one ``multimem.st`` per 16 bytes (the switch replicates), else one store per peer."""
        self.epoch += 1
        native().allgather_bf16([self.ws.data_ptr(p, self._param_off) for p in range(self.world)], self.rank,
                                bucket_numel, flat_param.numel(), self._flag_ptrs(), self.epoch, head, self._mc_param)
