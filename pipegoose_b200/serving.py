"""Continuous batching over a paged KV cache: requests join and leave a running batch independently.

    engine = ContinuousBatcher(model, max_cache_tokens=1 << 20)
    rid = engine.submit(prompt_ids, max_new_tokens=128)
    done = engine.step()     # [(rid, prompt + new tokens)] of the requests that finished in this step
    outs = engine.run()      # step until every submitted request is done -> {rid: tokens}

The engine owns the keys and values of every layer in two pools of 64-position pages, ``[n_layer, num_pages, n_head,
64, D]``, shared block tables for all layers and a free list.  A request is admitted first come, first served (no
request overtakes an earlier one) as soon as ``ceil((prompt + max_new_tokens) / 64)`` pages are free; they are reserved
until it finishes, so nothing is ever preempted, and return to the free list in the step it finishes.

A step is either one prefill of newly admitted prompts, packed into one row of at most ``max_prefill_tokens`` tokens
(a longer prompt runs alone) through the document-masked flash kernel, or one decode of every running sequence
through the paged split-KV decode kernel.  Tokens are chosen with the model's ``_select_token``, one call per group of
requests that share sampling parameters.  A step makes one host-to-device upload (tokens, positions and page tables,
shared by all layers) and one device-to-host transfer (the chosen tokens).

Limits: sampled tokens depend on which requests share a step (the random stream is consumed per group);
an ``ExpertLayer`` capacity limit counts the tokens of one step, as in ``generate()``.  Tensor-parallel, pipelined and
fused NVLink MoE models are refused.
"""
from __future__ import annotations

import collections
import itertools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from pipegoose_b200.ops.attention import PAGE_SIZE


@dataclass
class _Request:
    rid: int
    tokens: List[int]
    prompt_len: int
    max_new_tokens: int
    sampling: Tuple            # (do_sample, temperature, top_k, top_p): requests with the same tuple are picked together
    eos_token_id: Optional[int]
    pages: List[int] = field(default_factory=list)

    @property
    def pages_needed(self) -> int:
        return -(-(self.prompt_len + self.max_new_tokens) // PAGE_SIZE)


class ContinuousBatcher:
    """Continuous-batching generation for a ``BloomForCausalLM`` / ``GPT2LMHeadModel`` (module docstring).

    ``max_cache_tokens``: KV-cache positions the pools hold (rounded down to whole pages of 64).
    ``max_prefill_tokens``: most prompt tokens packed into one prefill step.
    ``generator``: random stream of sampled requests."""

    def __init__(self, model, max_cache_tokens: int, max_prefill_tokens: int = 8192,
                 generator: Optional[torch.Generator] = None):
        from pipegoose_b200.models.bloom import BloomMLP, _decodes_incrementally

        if getattr(model, "tp", None) is not None:
            raise ValueError("ContinuousBatcher serves single-GPU models: tensor-parallel models are not supported")
        if getattr(model, "_pg_pipeline_engine", None) is not None:
            raise ValueError("ContinuousBatcher serves single-GPU models: pipelined (PipelineParallel) models are not "
                             "supported")
        blocks = model.transformer.h
        if not all(isinstance(b.mlp, BloomMLP) or _decodes_incrementally(b.mlp) for b in blocks):
            raise ValueError("ContinuousBatcher does not support the fused NVLink MoE layer (its kernels are built "
                             "around token-sharded full sequences); use ExpertLayer MLPs")
        if max_prefill_tokens < 1:
            raise ValueError(f"max_prefill_tokens must be at least 1, got {max_prefill_tokens}")
        cfg = model.config
        self.model = model
        self.max_prefill_tokens = int(max_prefill_tokens)
        self.generator = generator
        self.num_pages = int(max_cache_tokens) // PAGE_SIZE
        if self.num_pages < 1:
            raise ValueError(f"max_cache_tokens = {max_cache_tokens} holds no page of {PAGE_SIZE} positions")
        self.n_positions = cfg.n_positions if getattr(cfg, "position_embedding", "alibi") == "learned" else None
        w = blocks[0].self_attention.query_key_value.weight
        D = cfg.hidden_size // cfg.n_head
        shape = (len(blocks), self.num_pages, cfg.n_head, PAGE_SIZE, D)
        self.k_pools = torch.empty(shape, dtype=w.dtype, device=w.device)
        self.v_pools = torch.empty(shape, dtype=w.dtype, device=w.device)
        self.device = w.device
        self._free = collections.deque(range(self.num_pages))
        self._ids = itertools.count()
        self._waiting: collections.deque = collections.deque()    # submitted, no pages yet
        self._admitted: collections.deque = collections.deque()   # pages reserved, prompt not yet run
        self._running: List[_Request] = []                        # prompt in the cache, decoding

    # ------------------------------------------------------------------ public
    def submit(self, prompt_ids: Sequence[int], max_new_tokens: int, do_sample: bool = False, temperature: float = 1.0,
               top_k: int = 0, top_p: float = 1.0, eos_token_id: Optional[int] = None) -> int:
        """Queue one request; returns its id.  The arguments mean what they mean in ``generate()``."""
        tokens = [int(t) for t in (prompt_ids.reshape(-1).tolist() if torch.is_tensor(prompt_ids) else prompt_ids)]
        if not tokens:
            raise ValueError("empty prompt: a request needs at least one token")
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be at least 1, got {max_new_tokens}")
        # the last new token is never fed back: positions 0 .. prompt + max_new_tokens - 2 are embedded
        if self.n_positions is not None and len(tokens) + max_new_tokens - 1 > self.n_positions:
            raise ValueError(f"prompt ({len(tokens)}) + max_new_tokens ({max_new_tokens}) - 1 positions exceed the "
                             f"model's n_positions = {self.n_positions}")
        r = _Request(next(self._ids), tokens, len(tokens), int(max_new_tokens),
                     (bool(do_sample), float(temperature), int(top_k), float(top_p)) if do_sample else (False,),
                     eos_token_id)
        if r.pages_needed > self.num_pages:
            raise ValueError(f"the request needs {r.pages_needed} pages of {PAGE_SIZE} positions (prompt {len(tokens)} + "
                             f"max_new_tokens {max_new_tokens}); the pool has {self.num_pages}")
        self._waiting.append(r)
        return r.rid

    def has_work(self) -> bool:
        return bool(self._waiting or self._admitted or self._running)

    def step(self) -> List[Tuple[int, List[int]]]:
        """One prefill or one decode step; returns ``(rid, prompt + new tokens)`` of the requests that finished."""
        self._admit()
        reqs, logits = self._forward()
        if not reqs:
            return []
        chosen = self._select(reqs, logits)
        done = []
        for r, t in zip(reqs, chosen):
            r.tokens.append(t)
            if len(r.tokens) - r.prompt_len == r.max_new_tokens or t == r.eos_token_id:
                self._free.extend(r.pages)
                r.pages = []
                done.append((r.rid, r.tokens))
            else:
                self._running.append(r)
        return done

    def run(self) -> Dict[int, List[int]]:
        """Step until every submitted request is done."""
        outs = {}
        while self.has_work():
            outs.update(self.step())
        return outs

    # ------------------------------------------------------------------ internals
    def _admit(self) -> None:
        while self._waiting and self._waiting[0].pages_needed <= len(self._free):
            r = self._waiting.popleft()
            r.pages = [self._free.popleft() for _ in range(r.pages_needed)]
            if not all(0 <= p < self.num_pages for p in r.pages):
                raise RuntimeError(f"page ids {r.pages} outside the pool of {self.num_pages} pages")
            self._admitted.append(r)

    def _upload(self, rows: List[List[int]]) -> List[torch.Tensor]:
        """Host int lists -> int32 device tensors, in one copy."""
        flat = torch.tensor(list(itertools.chain.from_iterable(rows)), dtype=torch.int32).to(self.device)
        return list(flat.split([len(r) for r in rows]))

    def _forward(self) -> Tuple[List[_Request], torch.Tensor]:
        """The requests this step serves, with requests that share sampling parameters adjacent, and their fp32
        next-token logits ``[len(reqs), V]``."""
        if self._admitted:                                      # prefill the oldest admitted prompts
            reqs, n = [], 0
            while self._admitted and (not reqs or n + self._admitted[0].prompt_len <= self.max_prefill_tokens):
                reqs.append(self._admitted.popleft())
                n += reqs[-1].prompt_len
            reqs.sort(key=lambda r: r.sampling)
            ids, positions, seg, slot, last, o = [], [], [], [], [], 0
            for r in reqs:
                P = r.prompt_len
                ids += r.tokens
                positions += range(P)
                seg += [o] * P
                slot += [r.pages[p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE for p in range(P)]
                o += P
                last.append(o - 1)
            ids, positions, seg, slot, last = self._upload([ids, positions, seg, slot, last])
            logits = self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, seg_start=seg, slot=slot,
                                              last=last)
            return reqs, logits.float()
        reqs = sorted(self._running, key=lambda r: r.sampling)
        self._running = []
        if not reqs:
            return [], None
        width = max(len(r.pages) for r in reqs)
        table = [p for r in reqs for p in r.pages + [0] * (width - len(r.pages))]
        pos = [len(r.tokens) - 1 for r in reqs]
        ids, positions, table = self._upload([[r.tokens[-1] for r in reqs], pos, table])
        logits = self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, table=table.view(len(reqs), width),
                                          max_pos=max(pos))
        return reqs, logits.float()

    def _select(self, reqs: List[_Request], logits: torch.Tensor) -> List[int]:
        """Next token of every request (``reqs`` grouped by sampling parameters), one device-to-host transfer."""
        picks, i = [], 0
        for key, group in itertools.groupby(reqs, key=lambda r: r.sampling):
            n = len(list(group))
            do_sample, temperature, top_k, top_p = key if key[0] else (False, 1.0, 0, 1.0)
            picks.append(self.model._select_token(logits[i:i + n], do_sample, temperature, top_k, top_p, self.generator))
            i += n
        return torch.cat(picks).tolist()
