"""Fused expert-parallel Switch MLP: router kernel, NVLink all-to-all dispatch fused with the token
permute, grouped wgmma expert GEMMs (chunk = expert, started per expert as soon as its tokens
landed), and combine fused into the last expert GEMM's epilogue (rows scaled by the gate weight and
stored straight into the source rank's buffer).

Layout: the experts of a layer are sharded over the EXPERT (== TENSOR) group, ``E_local`` per rank;
tokens are sharded over the same group (sequence-parallel activations ``[n, h]``).  Every
``(expert, source rank)`` pair owns a fixed window of ``C`` rows in the expert's input buffer, so
dispatch needs no count exchange and no host synchronisation; tokens beyond the window are dropped
(they pass through on the residual path), i.e. the Switch capacity limit is enforced per source
rank.  Buffers and arrival counters are double-buffered by call parity and reset after use.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.distributed as dist
from torch import nn

from pipegoose_b200.distributed import symmetric as S
from pipegoose_b200.distributed.parallel_mode import ParallelMode
from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops import native
from pipegoose_b200.ops.functional import _main_grad, acquire_main_grad, notify_grad_ready

SIG_MOE_FWD = 256   # [256, 256+E_local): arrival counters of forward dispatches
SIG_MOE_BWD = 320   # backward dispatches
DISPATCH_BLOCKS = 64


def _round_up(x, m):
    return (x + m - 1) // m * m


class MoEWorkspace:
    """Peer-mapped buffers of one EP group for one (n, h, E, K, capacity) configuration."""

    def __init__(self, ctx, mode, n, h, E_local, T, top_k, C):
        self.ctx, self.mode = ctx, mode
        self.n, self.h, self.E_local, self.T, self.K, self.C = n, h, E_local, T, top_k, C
        self.rank = ctx.get_local_rank(mode)
        self.rows = E_local * T * C
        xbytes = self.rows * h * 2
        meta = _round_up(self.rows * 4, 1024)
        comb = top_k * n * h * 2
        # per parity: [x rows | row_ret | row_scale | comb]
        self.slot_bytes = _round_up(xbytes + 2 * meta + comb, 1024)
        self.off_ret, self.off_scale, self.off_comb = xbytes, xbytes + meta, xbytes + 2 * meta
        # 2 parities x {fwd, bwd}
        self.ws = S.SymmetricWorkspace(ctx, mode, 4 * self.slot_bytes)
        self.calls = {"fwd": 0, "bwd": 0}
        for kind in ("fwd", "bwd"):
            for parity in (0, 1):
                self.reset(kind, parity)
        torch.cuda.synchronize()
        dist.barrier(group=ctx.get_group(mode))

    def _base(self, kind, parity):
        return ((0 if kind == "fwd" else 2) + parity) * self.slot_bytes

    def xbuf(self, kind, parity):
        return self.ws.local_tensor(self._base(kind, parity), (self.rows, self.h), torch.bfloat16)

    def row_ret(self, kind, parity):
        return self.ws.local_tensor(self._base(kind, parity) + self.off_ret, (self.rows,), torch.int32)

    def row_scale(self, kind, parity):
        return self.ws.local_tensor(self._base(kind, parity) + self.off_scale, (self.rows,), torch.float32)

    def comb(self, kind, parity):
        return self.ws.local_tensor(self._base(kind, parity) + self.off_comb, (self.K * self.n, self.h), torch.bfloat16)

    def peer(self, kind, parity, rank, off):
        return self.ws.data_ptr(rank, self._base(kind, parity) + off)

    def reset(self, kind, parity):
        self.xbuf(kind, parity).zero_()
        self.row_ret(kind, parity).fill_(-1)
        self.row_scale(kind, parity).fill_(1.0)
        self.comb(kind, parity).zero_()

    def close(self):
        self.ws.close()


class _FusedMoE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, wg, bg, w1, b1, w2, b2, layer):
        eng: MoEWorkspace = layer._workspace(x.shape[0], x.shape[1])
        n, h = x.shape
        E, K_, T, El, C = layer.num_experts, layer.top_k, eng.T, eng.E_local, eng.C
        dev = x.device
        probs = torch.empty(n, E, dtype=torch.float32, device=dev)
        lse = torch.empty(n, dtype=torch.float32, device=dev)
        topk_idx = torch.empty(n, K_, dtype=torch.int32, device=dev)
        topk_prob = torch.empty(n, K_, dtype=torch.float32, device=dev)
        pos = torch.empty(n, K_, dtype=torch.int32, device=dev)
        counts = torch.zeros(E, dtype=torch.int32, device=dev)
        prob_sum = torch.zeros(E, dtype=torch.float32, device=dev)
        zsum = torch.zeros(1, dtype=torch.float32, device=dev)
        jitter = None
        if layer.training and layer.jitter_eps > 0:
            jitter = torch.rand(n, E, device=dev) * (2 * layer.jitter_eps) + (1 - layer.jitter_eps)
        x = x.contiguous()
        native().moe_route(x, wg, bg, jitter, K_, C, probs, topk_idx, topk_prob, pos, counts, prob_sum, zsum, lse)

        eng.calls["fwd"] += 1
        call = eng.calls["fwd"]
        par = call & 1
        peers = range(T)
        native().moe_dispatch(x, topk_idx, topk_prob, pos,
                              [eng.peer("fwd", par, p, 0) for p in peers],
                              [eng.peer("fwd", par, p, eng.off_ret) for p in peers],
                              [eng.peer("fwd", par, p, eng.off_scale) for p in peers],
                              [eng.ws.sig_ptr(p, SIG_MOE_FWD) for p in peers], K_, El, C, eng.rank, False, DISPATCH_BLOCKS)
        xbuf = eng.xbuf("fwd", par)
        rows = eng.rows
        f = w1.shape[1]  # 4h
        z = torch.empty(rows, f, dtype=torch.bfloat16, device=dev)
        h1 = torch.empty(rows, f, dtype=torch.bfloat16, device=dev)
        # grouped fc1 (+bias +GELU): chunk e waits for its T*DISPATCH_BLOCKS arrivals
        native().gemm(xbuf, w1.view(El * f, h), h1, False, False, b1.view(-1), None, z, K.EPI_GELU, 0, 0,
                      El, 0, eng.ws.sig_ptr(eng.rank, SIG_MOE_FWD), T * DISPATCH_BLOCKS * call, [], [],
                      dict(b_chunk_rows=f, bias_chunk_stride=f))
        x_saved = xbuf.clone()
        ret = eng.row_ret("fwd", par)
        scale = eng.row_scale("fwd", par)
        ret_saved, scale_saved = ret.clone(), scale.clone()
        # grouped fc2 (+bias), combine in the epilogue: row -> source rank's comb[k*n + token], scaled by the gate prob
        dummy = layer._dummy(h, dev)
        native().gemm(h1, w2.view(El * h, f), dummy, False, False, b2.view(-1), None, None, K.EPI_SCATTER, 0, 0,
                      El, 0, 0, 0, [eng.peer("fwd", par, p, eng.off_comb) for p in peers], [],
                      dict(b_chunk_rows=h, bias_chunk_stride=h, row_ret=ret.data_ptr(), row_scale=scale.data_ptr(), rows_per_src=C))
        layer._barrier(eng)
        comb = eng.comb("fwd", par)
        y = torch.empty(n, h, dtype=torch.bfloat16, device=dev)
        native().rs_reduce(comb.data_ptr(), K_, n * h, eng.ws.sig_ptr(eng.rank, S.SIG_BARRIER), 0, None, residual, y)
        comb_saved = comb.clone()
        eng.reset("fwd", par)  # stream-ordered after the consumers above; peers reuse this parity two calls later
        ctx.save_for_backward(x, wg, bg, w1, b1, w2, b2, probs, topk_idx, topk_prob, pos, x_saved, z, h1,
                              ret_saved, scale_saved, comb_saved, jitter if jitter is not None else torch.empty(0, device=dev),
                              lse)
        ctx.layer = layer
        n_f = float(n)
        # Switch load-balancing loss alpha * E * <tokens per expert, mean prob per expert>; z-loss mean(lse^2)
        aux = layer.alpha * E * torch.sum((counts.float() / n_f) * (prob_sum / n_f))
        zl = zsum[0] / n_f
        ctx.aux_coeff = layer.alpha * E * counts.float() / n_f / n_f  # d aux / d probs[t, e]
        return y, aux, zl, probs, lse

    @staticmethod
    def backward(ctx, dy, daux, dz_loss, dprobs_ext, dlse_ext):
        (x, wg, bg, w1, b1, w2, b2, probs, topk_idx, topk_prob, pos, x_saved, z, h1, ret_saved, scale_saved,
         comb_saved, jitter, lse) = ctx.saved_tensors
        layer = ctx.layer
        n, h = x.shape
        eng: MoEWorkspace = layer._workspace(n, h)
        E, K_, T, El, C = layer.num_experts, layer.top_k, eng.T, eng.E_local, eng.C
        dev = x.device
        f = w1.shape[1]
        dy = dy.contiguous()
        rows = eng.rows
        # ---- gate-weight gradient from the combine: d p_k[t] = <expert_out_k[t], dy[t]> = <comb_k[t], dy[t]> / p_k[t]
        dots = (comb_saved.view(K_, n, h).float() * dy.float().unsqueeze(0)).sum(-1).t()  # [n, K]
        dp_topk = torch.where(pos >= 0, dots / topk_prob.clamp_min(1e-20), torch.zeros_like(dots))
        # ---- dispatch p * dy to the experts
        eng.calls["bwd"] += 1
        call = eng.calls["bwd"]
        par = call & 1
        peers = range(T)
        native().moe_dispatch(dy, topk_idx, topk_prob, pos,
                              [eng.peer("bwd", par, p, 0) for p in peers],
                              [eng.peer("bwd", par, p, eng.off_ret) for p in peers],
                              [eng.peer("bwd", par, p, eng.off_scale) for p in peers],
                              [eng.ws.sig_ptr(p, SIG_MOE_BWD) for p in peers], K_, El, C, eng.rank, True, DISPATCH_BLOCKS)
        dybuf = eng.xbuf("bwd", par)
        # grouped dgrad through fc2 with GELU' epilogue: dz = (dyb @ W2) * gelu'(z); waits per expert for arrivals
        dz = torch.empty(rows, f, dtype=torch.bfloat16, device=dev)
        native().gemm(dybuf, w2.view(El * h, f), dz, False, True, None, None, z, K.EPI_DGELU, 0, 0,
                      El, 0, eng.ws.sig_ptr(eng.rank, SIG_MOE_BWD), T * DISPATCH_BLOCKS * call, [], [],
                      dict(b_chunk_rows=h))
        dyb = dybuf.clone()
        # grouped dgrad through fc1, combined straight back into the source ranks' dx buffers (scale 1)
        ones = layer._ones(rows, dev)
        native().gemm(dz, w1.view(El * f, h), layer._dummy(h, dev), False, True, None, None, None, K.EPI_SCATTER, 0, 0,
                      El, 0, 0, 0, [eng.peer("bwd", par, p, eng.off_comb) for p in peers], [],
                      dict(b_chunk_rows=f, row_ret=ret_saved.data_ptr(), row_scale=ones.data_ptr(), rows_per_src=C))
        # per-expert weight gradients (contraction over the expert's row window)
        R = T * C
        dw1 = torch.empty_like(w1) if _main_grad(w1) is None else None
        dw2 = torch.empty_like(w2) if _main_grad(w2) is None else None
        db1 = torch.empty_like(b1) if _main_grad(b1) is None else None
        db2 = torch.empty_like(b2) if _main_grad(b2) is None else None
        mg = {}
        for name, p in (("w1", w1), ("w2", w2)):
            if _main_grad(p) is not None:
                mg[name] = acquire_main_grad(p, will_overwrite=True)
        for name, p in (("b1", b1), ("b2", b2)):
            if _main_grad(p) is not None:
                mg[name] = acquire_main_grad(p, will_overwrite=False)
        for e in range(El):
            sl = slice(e * R, (e + 1) * R)
            if dw2 is None:
                K.gemm_tn(dyb[sl], h1[sl], accum_into=mg["w2"][0][e], accumulate=mg["w2"][1])
                K.gemm_tn(dz[sl], x_saved[sl], accum_into=mg["w1"][0][e], accumulate=mg["w1"][1])
            else:
                dw2[e] = K.gemm_tn(dyb[sl], h1[sl])
                dw1[e] = K.gemm_tn(dz[sl], x_saved[sl])
            if db2 is None:
                K.colsum(dyb[sl], accum_into=mg["b2"][0][e])
                K.colsum(dz[sl], accum_into=mg["b1"][0][e])
            else:
                db2[e] = K.colsum(dyb[sl])
                db1[e] = K.colsum(dz[sl])
        for p in (w1, w2, b1, b2):
            if _main_grad(p) is not None:
                notify_grad_ready(p)
        layer._barrier(eng)
        dcomb = eng.comb("bwd", par)
        dx = torch.empty(n, h, dtype=torch.bfloat16, device=dev)
        native().rs_reduce(dcomb.data_ptr(), K_, n * h, eng.ws.sig_ptr(eng.rank, S.SIG_BARRIER), 0, None, None, dx)
        eng.reset("bwd", par)
        # ---- router backward (tiny: [n, E]); fp32 math with torch
        dprobs = torch.zeros_like(probs)
        dprobs.scatter_add_(1, topk_idx.long(), dp_topk)
        if daux is not None:
            dprobs = dprobs + daux * ctx.aux_coeff.unsqueeze(0)
        if dprobs_ext is not None:
            dprobs = dprobs + dprobs_ext
        dlogits = probs * (dprobs - (probs * dprobs).sum(-1, keepdim=True))
        lse_grad = torch.zeros(n, device=dev)
        if dz_loss is not None:
            lse_grad = lse_grad + dz_loss * 2.0 * lse / n
        if dlse_ext is not None:
            lse_grad = lse_grad + dlse_ext
        dlogits = dlogits + lse_grad.unsqueeze(-1) * probs
        if jitter.numel() > 0:
            dlogits = dlogits * jitter
        dx = dx + (dlogits.to(torch.bfloat16) @ wg)
        dwg = (dlogits.t() @ x.float()).to(wg.dtype)
        dbg = dlogits.sum(0).to(bg.dtype) if bg is not None else None
        return dx, dy, dwg, dbg, dw1, db1, dw2, db2, None


class FusedExpertLayer(nn.Module):
    """Drop-in for a Bloom block's MLP (``forward(layernorm_output, residual)``) on the fused MoE path."""

    def __init__(self, num_experts: int, expert: nn.Module, router: nn.Module, parallel_context, top_k: Optional[int] = None,
                 capacity_factor: float = 1.25, parallel_mode: ParallelMode = ParallelMode.TENSOR):
        super().__init__()
        self.parallel_context = parallel_context
        self.parallel_mode = parallel_mode
        T = parallel_context.get_world_size(parallel_mode)
        assert num_experts % T == 0
        self.num_experts = num_experts
        self.num_local_experts = num_experts // T
        self.router = router
        self.top_k = top_k if top_k is not None else getattr(router, "top_k", 1)
        self.alpha = getattr(router, "alpha", 0.01)
        noise = getattr(router, "noise_policy", None)
        self.jitter_eps = getattr(noise, "eps", 0.0) if noise is not None else 0.0
        cap = getattr(router, "expert_capacity", None)
        self.capacity_factor = cap[0] if cap is not None else capacity_factor
        El = self.num_local_experts
        w1, b1 = expert.dense_h_to_4h.weight.data, expert.dense_h_to_4h.bias.data
        w2, b2 = expert.dense_4h_to_h.weight.data, expert.dense_4h_to_h.bias.data
        self.w1 = nn.Parameter(w1.unsqueeze(0).repeat(El, 1, 1).contiguous())
        self.b1 = nn.Parameter(b1.unsqueeze(0).repeat(El, 1).contiguous())
        self.w2 = nn.Parameter(w2.unsqueeze(0).repeat(El, 1, 1).contiguous())
        self.b2 = nn.Parameter(b2.unsqueeze(0).repeat(El, 1).contiguous())
        for p in (self.w1, self.b1, self.w2, self.b2):
            p.is_expert = True
        for p in self.router.parameters():
            p.tp_partial_grad = True  # gate gradients are partial sums over the token shards
        self._ws = {}
        self._tmp = {}
        self._barrier_epoch = 0

    # ------------------------------------------------------------------ helpers
    def _workspace(self, n, h) -> MoEWorkspace:
        key = (n, h)
        ws = self._ws.get(key)
        if ws is None:
            T = self.parallel_context.get_world_size(self.parallel_mode)
            per_src = math.ceil(self.capacity_factor * n * self.top_k / self.num_experts)
            C = _round_up(max(per_src, 1), max(128 // T, 1))
            while (T * C) % 128 != 0:
                C += 1
            ws = MoEWorkspace(self.parallel_context, self.parallel_mode, n, h, self.num_local_experts, T, self.top_k, C)
            self._ws[key] = ws
        return ws

    def _dummy(self, h, dev):
        t = self._tmp.get(("dummy", h))
        if t is None:
            t = self._tmp[("dummy", h)] = torch.empty(1, h, dtype=torch.bfloat16, device=dev)
        return t

    def _ones(self, rows, dev):
        t = self._tmp.get(("ones", rows))
        if t is None:
            t = self._tmp[("ones", rows)] = torch.ones(rows, dtype=torch.float32, device=dev)
        return t

    def _barrier(self, eng: MoEWorkspace):
        """All ranks' peer stores of this step are complete and visible."""
        self._barrier_epoch += 1
        key = id(eng)
        eng._bepoch = getattr(eng, "_bepoch", 0) + 1
        native().barrier_peers([eng.ws.sig_ptr(p, S.SIG_BARRIER) for p in range(eng.T)], eng.rank, eng._bepoch)

    @torch.no_grad()
    def to_expert_layer(self):
        """The same layer as a plain ``ExpertLayer`` (per-expert ``BloomMLP`` modules holding this rank's slices of the
        stacked weights, the same router object) — the form ``ExpertParallel.deparallelize`` and checkpoint export use."""
        from types import SimpleNamespace

        from pipegoose_b200.models.bloom import BloomMLP
        from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer

        h = self.w1.shape[2]
        template = BloomMLP(SimpleNamespace(hidden_size=h)).to(device=self.w1.device, dtype=self.w1.dtype)
        layer = ExpertLayer(self.num_experts, template, self.router, False, self.parallel_context)
        for j, expert in enumerate(layer.experts):
            expert.dense_h_to_4h.weight.copy_(self.w1[j])
            expert.dense_h_to_4h.bias.copy_(self.b1[j])
            expert.dense_4h_to_h.weight.copy_(self.w2[j])
            expert.dense_4h_to_h.bias.copy_(self.b2[j])
        for p in self.router.parameters():
            if hasattr(p, "tp_partial_grad"):
                del p.tp_partial_grad   # replicated tokens: the gate gradient is complete on every rank
        layer.train(self.training)
        return layer

    # ------------------------------------------------------------------ forward
    def forward(self, hidden_states: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        from pipegoose_b200.nn.expert_parallel.expert_context import ExpertContext

        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        res = residual.reshape(-1, shape[-1])
        gate = self.router.gate
        y, aux, zl, _probs, _lse = _FusedMoE.apply(x, res, gate.weight, gate.bias, self.w1, self.b1, self.w2, self.b2, self)
        # every rank of the group adds its (local-token) router losses to its loss while the gate's gradients are summed
        # over the group: 1/T of the gradient per rank keeps the objective's weight independent of the group size
        from pipegoose_b200.nn.expert_parallel.layers import _scale_grad

        T = self.parallel_context.get_world_size(self.parallel_mode)
        ectx = ExpertContext.get_instance()
        ectx.push_aux_loss(_scale_grad(aux, 1.0 / T))
        ectx.push_z_loss(_scale_grad(zl, 1.0 / T))
        return y.view(shape)
