"""Flat parameter / gradient storage.

``FlatModelState`` re-points every parameter of a module at a view of ONE contiguous buffer of
the model dtype and gives every parameter an fp32 ``main_grad`` view of ONE contiguous gradient
buffer.  That layout is what the GPU path is built around:

* the wgrad GEMM epilogue accumulates straight into ``param.main_grad`` (no ``.grad`` tensors,
  no bf16->fp32 cast pass);
* the data-parallel reducer walks the gradient buffer in fixed-size buckets (NVLink peer
  reduce-scatter/all-reduce kernels need contiguous, 16-byte aligned ranges);
* the ZeRO-1 optimizer owns a contiguous ``1/dp`` slice of the buffer and updates it with one
  fused Adam launch, then all-gathers the bf16 parameter buffer.

(The reference's ``Bucket`` re-points ``tensor.data`` the same way, core/bucket/bucket.py:52-54,
but nothing in the reference uses it.)
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Tuple

import torch
from torch import nn

_ALIGN = 128  # elements; keeps every view 256B-aligned for bf16 and 512B for fp32


def unique_parameters(module_or_params) -> List[nn.Parameter]:
    params = module_or_params.parameters() if isinstance(module_or_params, nn.Module) else module_or_params
    seen, out = set(), []
    for p in params:
        if id(p) not in seen and p.requires_grad:
            seen.add(id(p))
            out.append(p)
    return out


class FlatModelState:
    def __init__(self, params: Iterable[nn.Parameter], pad_to_multiple_of: int = 1, grad_dtype=torch.float32,
                 buffer_factory=None):
        self.params: List[nn.Parameter] = unique_parameters(list(params))
        assert len(self.params) > 0
        # parameters whose gradients are partial sums over the tensor-parallel group (sequence-parallel
        # LayerNorms / row-parallel biases) come first, contiguously: ONE all-reduce of flat_grad[:n] sums them
        # ... then the other small (< 2-D) parameters, then the matrices: [matrix_start, numel) holds only >= 2-D
        # parameters with complete gradients — the region the fused ZeRO-1 path reduce-scatters inside the kernels that
        # produce the gradients (wgrad epilogue, embedding backward), while [0, matrix_start) stays bucket-reduced
        self.params.sort(key=lambda p: 0 if getattr(p, "tp_partial_grad", False) else (1 if p.dim() < 2 else 2))  # stable
        self.tp_partial_numel = 0
        self.matrix_start = None
        self.inline = None    # the engine that reduce-scatters [matrix_start, numel) in-kernel (ops.comm.FusedDPEngine)
        p0 = self.params[0]
        self.device, self.dtype = p0.device, p0.dtype
        assert all(p.device == self.device and p.dtype == self.dtype for p in self.params), \
            "all parameters of a flat state must share device and dtype"
        self.offsets: Dict[int, Tuple[int, int]] = {}
        off = 0
        region_mult = max(pad_to_multiple_of, 1) * _ALIGN
        for p in self.params:
            if self.matrix_start is None and p.dim() >= 2 and not getattr(p, "tp_partial_grad", False):
                off = (off + region_mult - 1) // region_mult * region_mult   # slices of both regions stay aligned
                self.matrix_start = off
            self.offsets[id(p)] = (off, p.numel())
            off += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
            if getattr(p, "tp_partial_grad", False):
                self.tp_partial_numel = off
        mult = max(pad_to_multiple_of, 1) * _ALIGN
        self.numel = (off + mult - 1) // mult * mult
        if self.matrix_start is None:
            self.matrix_start = self.numel
        if buffer_factory is not None:
            # externally owned storage (NVLink peer-mapped symmetric memory for the fused DP/ZeRO kernels)
            self.flat_param, self.flat_grad = buffer_factory(self.numel, self.dtype, grad_dtype)
            self.flat_param.zero_(), self.flat_grad.zero_()
        else:
            self.flat_param = torch.zeros(self.numel, dtype=self.dtype, device=self.device)
            self.flat_grad = torch.zeros(self.numel, dtype=grad_dtype, device=self.device)
        for p in self.params:
            o, n = self.offsets[id(p)]
            view = self.flat_param[o:o + n].view_as(p.data)
            view.copy_(p.data)
            p.data = view
            p.main_grad = self.flat_grad[o:o + n].view_as(p.data)
            p._pg_flat_state = self
            p._mg_fresh = False
            p.grad = None
        self.begin_grad_window()

    @classmethod
    def of(cls, module: nn.Module, **kw) -> "FlatModelState":
        state = getattr(module, "_flat_state", None)
        if state is None:
            state = cls.find(module.parameters())
            if state is None:
                state = cls(module.parameters(), **kw)
            else:
                mult = max(kw.get("pad_to_multiple_of", 1), 1) * _ALIGN
                assert state.numel % mult == 0, "existing flat state is not padded for this data parallel size"
            module._flat_state = state
        return state

    @staticmethod
    def find(params) -> Optional["FlatModelState"]:
        """The flat state the given parameters already live in, if any."""
        for p in params:
            st = getattr(p, "_pg_flat_state", None)
            if st is not None:
                return st
        return None

    def zero_grad(self, lazy: bool = True):
        """Reset gradients.  ``lazy``: matrices are not memset — the first wgrad GEMM of the step
        overwrites instead of accumulating (``param._mg_fresh``); only the small 1-D parameters,
        whose gradients are built with atomics, are cleared here."""
        if getattr(self, "hold_grads", False):
            # produced by a pipeline schedule inside forward; the caller's ``loss.backward()`` has not run yet: this is the
            # ``zero_grad()`` of the canonical loop (forward, zero_grad, backward, step) and must not drop them
            return
        self.clears = getattr(self, "clears", 0) + 1    # (pipeline engines: a schedule after a real clear starts afresh)
        self.grads_materialized = False
        self.begin_grad_window()
        if self.inline is not None:
            # [matrix_start, numel) is reduce-scattered in-kernel: its owner slices are cleared by the optimizer step that
            # consumes them; an explicit clear (gradients produced but never consumed) is a collective: memset + peer barrier
            self.inline.clear_inline_region(force=not lazy)
        if not lazy:
            (self.flat_grad if self.inline is None else self.flat_grad[:self.matrix_start]).zero_()
            for p in self.params:
                p._mg_fresh = False
            return
        small = getattr(self, "_small_grads", None)
        if small is None:
            small = self._small_grads = [p.main_grad for p in self.params if p.dim() < 2]
        if small:
            torch._foreach_zero_(small)  # one multi-tensor launch instead of one fill per bias / LN vector
        inline_from = self.matrix_start if self.inline is not None else self.numel
        for p in self.params:
            p._mg_fresh = p.dim() >= 2 and self.offsets[id(p)][0] < inline_from

    def begin_grad_window(self):
        """The gradients of the previous window were consumed (optimizer step) or dropped (``zero_grad``): the next
        synced backward is the first reduction of a new window.  The gradient reducers use this to keep a second synced
        backward in ONE window correct (tensor-group SUM of partial gradients is not idempotent) or to refuse it
        (ZeRO-1 reduce-scatter)."""
        self.tp_reduced_base = None      # value of flat_grad[:tp_partial_numel] right after its last tensor-group sum
        self.reduced_in_window = False   # a data-parallel reduction already ran in this window

    def finalize_grads(self):
        """Parameters that received no gradient this step (still fresh) must read as zero."""
        for p in self.params:
            if getattr(p, "_mg_fresh", False):
                p.main_grad.zero_()
                p._mg_fresh = False

    def param_range(self, p: nn.Parameter) -> Tuple[int, int]:
        return self.offsets[id(p)]

    def shard_range(self, rank: int, world: int) -> Tuple[int, int]:
        assert self.numel % world == 0
        n = self.numel // world
        return rank * n, (rank + 1) * n

    def materialize_grads(self):
        """Hand the (reduced) fp32 main grads to a stock torch optimizer as ``.grad`` in the parameter dtype — always a
        COPY, added to a ``.grad`` that is already there (DDP semantics: several synced backward passes of one step
        accumulate) — and start a new gradient window: a bare ``torch.optim`` optimizer never calls
        :meth:`zero_grad` of this flat state, so the next backward must overwrite the main grads, not add to them."""
        self.grads_materialized = True
        for p in self.params:
            g = p.main_grad.to(p.dtype, copy=True)
            if p.grad is None:
                p.grad = g
            else:
                p.grad.add_(g)
            p._pg_materialized = p.grad   # (a copy of reduced main grads, not a gradient autograd delivered)
            p._mg_fresh = True
        self.begin_grad_window()

    def rebind(self):
        """Re-point the parameters after the module was moved (``.to`` creates new storages)."""
        for p in self.params:
            o, n = self.offsets[id(p)]
            if p.data.data_ptr() != self.flat_param[o:o + n].data_ptr():
                self.flat_param[o:o + n].view_as(p.data).copy_(p.data)
                p.data = self.flat_param[o:o + n].view_as(p.data)
