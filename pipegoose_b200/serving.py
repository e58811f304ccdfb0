"""Continuous batching over a paged KV cache: requests join and leave a running batch independently.

    engine = ContinuousBatcher(model, max_cache_tokens=1 << 20)
    rid = engine.submit(prompt_ids, max_new_tokens=128)
    done = engine.step()     # [(rid, prompt + new tokens)] of the requests that finished in this step
    outs = engine.run()      # step until every submitted request is done -> {rid: tokens}

The engine owns the keys and values of every layer in two pools of 64-position pages, ``[n_layer, num_pages, n_head,
64, D]``, shared block tables for all layers and a free list.  A request is admitted first come, first served (no
request overtakes an earlier one) as soon as ``ceil((prompt + max_new_tokens) / 64)`` pages are free; they are reserved
until it finishes, so nothing is ever preempted (unless ``preemption=True``: below), and return to the free list in the
step it finishes.

A step is either one prefill of newly admitted prompts, packed into one row of at most ``max_prefill_tokens`` tokens
(a longer prompt runs alone) through the document-masked flash kernel, or one decode of every running sequence
through the paged split-KV decode kernel (or, with speculative decoding, a verify step; with chunked prefill, a mixed
step: below).  Tokens are chosen with the model's ``_select_token``, one call per group of
requests that share sampling parameters.  A step makes one host-to-device upload (tokens, positions and page tables,
shared by all layers) and one device-to-host transfer (the chosen tokens).

Prefix caching (``prefix_caching=True``, off by default): full pages of prompts (and, once a request finishes, of its
generated tokens) stay indexed by their content after use, so a later prompt that starts with the same tokens reuses
them instead of computing them again.  The key of page k of a sequence is (key id of page k-1, its 64 token ids):
matching compares token ids exactly.  A request matches its prompt page by page, at most ``(prompt - 1) // 64`` pages
(its last prompt token is always computed: the step needs its logits), and takes a reference on every hit.  Pages are
reference-counted; at zero a page returns to the free list but keeps its index entry until it is handed out again,
least recently freed first (a finished request releases its last page first, so a chain's tail is evicted before its
prefix).  Invariant: only full pages are shared, and a request never writes into a shared page (its first computed
position is a page boundary, and decoding writes past the prompt), so no page is ever copied.  A prefill step in which
some request has a hit runs every request through the paged prefill kernel over the pools (a request without one
from position 0); otherwise the flash-kernel path above runs.  ``cached_prompt_tokens`` counts the prompt tokens served
from the cache.  With prefix caching a request's tokens can depend, at rounding level, on which earlier requests left
pages behind.

FP8 KV cache (``kv_cache_dtype=torch.float8_e4m3fn``, off by default): the pools hold one ``float8_e4m3fn`` code per
element, with fp32 scales ``k_scales`` / ``v_scales [n_layer, num_pages, n_head, 64]``, one per position and head
(``ops.attention.quantize_kv`` is the format).  The same memory holds about 1.9x the positions.  A step's queries read
positions computed in earlier steps from the FP8 pools, dequantized, and positions computed in the same step from
that step's bf16 ``qkv``, exactly.  So a prefill without prefix hits gives the same logits as with default pools (the
flash kernel runs on ``qkv``; only the cache write quantizes), and a decode step reads its own key exactly.  A
prefill with hits dequantizes the sequences' cached pages into a bf16 staging pool sized for the step's prompt pages
and runs the paged prefill kernel on it.  A scale belongs to its page slot, so prefix sharing, reference counting and
eviction are unchanged.  Accuracy on trained checkpoints is not verified here.

Chunked prefill (``chunked_prefill=True``, off by default): a step then carries one decode token of every running
request and, after them, chunks of admitted prompts, taken first come, first served until the step holds
``max_prefill_tokens`` prompt tokens (decode tokens do not count).  A chunk that does not end its prompt ends on a page
boundary, so every chunk starts on one (a prefix-cache start is one too), and the rest of that prompt waits for the
next step; ``max_prefill_tokens`` must be at least 64.  The decode rows go through the paged decode kernel and the
chunks through the paged prefill kernel over the pools (over FP8 pools through a staging pool of the chunks' pages, as
a prefill with hits), in one forward; they write disjoint pages.  A request whose
prompt completes chooses its first token in that step and decodes from the next; only then are its pages indexed and
its ``cached`` counted in ``cached_prompt_tokens``.  A step without admitted prompts is the decode step above, and a step
without running requests carries only chunks.  So a long prompt delays the running requests by one bounded step at a
time instead of its whole prefill.  With FP8 pools a chunk reads the earlier chunks of its prompt from the pools,
dequantized (positions computed in earlier steps), so a chunked prompt's logits differ from those of an unchunked
prefill by the FP8 rounding of those keys and values.  Refused with speculative decoding.

Speculative decoding (``num_speculative_tokens=k``, 0 .. 7, off by default; refused with FP8 pools): before a decode
step every running request drafts up to k tokens by prompt lookup, the tokens that followed the most recent earlier
occurrence of its last ``SPEC_NGRAM_SIZES`` = 3 (else 2) tokens, found in a per-request n-gram index updated with
each new token.  A draft never exceeds ``max_new_tokens - generated - 1`` tokens, so the step writes only inside the
pages reserved at admission.  If no request has a draft, the step is the decode step above.  Otherwise it is a verify
step: every running request appends its last token and its drafts (one token without a draft) through the paged
append-attention kernel, which writes their keys and values and returns the logits of every token; each request
keeps the drafts ``verify_drafts`` accepts plus one more token, cut at ``eos_token_id`` and ``max_new_tokens``.
Greedy requests accept a draft while it is the arg-max; sampled requests use rejection sampling, which keeps the
distribution of non-speculative sampling.  Still one upload and one device-to-host transfer per step.  Invariant:
positions ``0 .. len(tokens) - 2`` of a request are always valid in its pages.  Rejected drafts leave stale keys and
values behind the accepted ones; the next step of that request writes those positions before any query reads them,
and ``_release`` indexes only the valid positions.  ``speculative_proposed_tokens`` counts the drafts verified and
``speculative_accepted_tokens`` the accepted drafts that were emitted (not those cut off after an eos).

CUDA graphs (``cuda_graphs=True``, off by default): the plain decode step (one token per running request through the
paged decode kernel, in every mode above: the decode steps of the default engine, steps without chunks under chunked
prefill, steps without drafts under speculative decoding, and over FP8 pools) is replayed from a CUDA graph instead of
being issued op by op from Python.  Prefill steps (with or without cached prefixes), mixed steps and verify steps stay
eager.  A step with B running requests replays the graph of the smallest of ``GRAPH_BATCH_SIZES`` that holds B; a
larger step runs eager.  A bucket's graph is captured on the first step that needs it (after one eager warm-up call
on the capture stream) and kept for the engine's lifetime; all graphs share one memory pool.  Every graph reads one
static int32 buffer (ids, positions, and page tables of one width W, the most pages one request can reserve), filled
from a pinned host mirror by one copy per step, and is captured with ``max_pos = W * 64 - 1``, which only shapes the
kernel's grid.  Rows past B are padding: token 0 at position 0 over a table row of the scratch page, one extra page
(index ``num_pages``) of every pool and scale pool that never enters the free list.  The graph writes the logits into
a static ``[bucket, V]`` buffer and token choice runs eagerly on its first B rows, so it is the eager engine's choice
for the same logits.  A bucket's kernel grid, and cuBLAS's choice for the padded M, can differ from the eager step's,
so logits can differ from the eager engine's at rounding level.  Costs: the graphs' pool (the largest bucket's logits
alone are 256 x V model-dtype values) and a capture pause the first time a bucket is used.  Needs the native decode
path (CUDA bf16 weights, head size 64, 80 or 128) and ``BloomMLP`` MLPs (``ExpertLayer`` routing depends on the data):
refused otherwise.  ``graph_decode_steps`` counts the decode steps served by a replay.

Beam search (``submit(..., num_beams=W)``, 2 .. ``MAX_BEAMS`` = 8; ``num_beams=1`` is the plain request): 🤗's
``GenerationMixin._beam_search`` per request, with ``length_penalty``, ``early_stopping`` (True, False or "never") and
``num_return_sequences``.  Every step keeps the 2W best candidates over the request's W beams (its first step: 2W from
the prompt's one row), sends those among the top W that end in ``eos_token_id`` (or reach ``max_new_tokens``) to the
finished hypotheses with the length penalty on the generated length, continues with the W best of the others and stops
by 🤗's rules.  The result is the best hypothesis; ``hypotheses[rid]`` holds the ``num_return_sequences`` best
``(prompt + tokens, score)``, best first, with 🤗's ``sequences_scores`` as score, and the caller pops its entries.
The beams are decode rows like any request's, through the paged decode kernel, in mixed steps and in graph replays
(whose buckets count rows); the beam step runs eagerly after the forward, on the model-dtype logits, through one
``beam_topk`` call (a fused log-softmax and top-k) for all beam requests and one device-to-host transfer.
Reservation: a beam request reserves ``prompt // 64 + W * (pages - prompt // 64)`` pages at admission (the prompt's
full pages once, the rest per beam) and is admitted, and releases every page, like any request, so nothing is ever
preempted; ``submit`` refuses it if that exceeds the pool.  Forks: inside the request its reserved pages are shared out
among its beams with request-local reference counts.  After a beam step every new beam takes its parent's page list
(references are taken before the old beams' are dropped).  Copy-on-write: the page holding a beam's next write
position ``len(tokens) - 1`` must be that beam's alone; the first of its holders in 🤗's order keeps it, every other
gets a page from the request's reserve with the leading ``pos % 64`` slots copied, and at ``pos % 64 == 0`` the write
starts a fresh page.  One ``paged_kv_copy`` launch per step copies every such page in every layer (with its scales
over FP8 pools); ``beam_page_copies`` counts them.  A request that would need more pages than it reserved raises
``RuntimeError``.  With prefix caching a beam request takes its prompt's hits as any request does and indexes its
prompt's pages only, never beam pages.  Beam requests work with prefix caching, FP8 pools, chunked prefill and
``cuda_graphs``, beside greedy and sampled requests, whose tokens do not depend on them (up to the rounding a graph
bucket or cuBLAS's choice for another M brings, as above).  Refused: ``num_beams`` outside 1 .. 8, ``do_sample=True``
with ``num_beams > 1`` (beam sampling), ``num_return_sequences`` outside 1 .. ``num_beams``, ``2 * num_beams`` above the
vocabulary, and beam requests on an engine with speculative decoding.

Preemption (``preemption=True``, off by default; ``swap_space_tokens`` sizes a pinned host pool of whole pages and
needs it): plain requests take pages as they grow instead of reserving their whole length.  A request is admitted with
the pages of its tokens so far (minus prefix hits); before every decode, mixed or verify step each running plain
request whose next write starts a page takes one off the free list.  So a request that stops at ``eos_token_id`` early
never held the pages it did not write, and the pool holds more running requests.  When the free list cannot cover a
step's growth, running plain requests are preempted, latest submitted first, until it can (a request may preempt
itself; ``submit`` still refuses a request longer than the pool, so the oldest can always finish).  A victim whose pages
fit in the free host slots is swapped out: one ``paged_kv_swap`` per step copies every such victim's pages, every layer,
K and V (codes and scales over FP8 pools), to the host pool, and its pages are freed.  Otherwise it is recomputed: its
pages are freed (with prefix caching ``_release`` indexes its full pages first, so its readmission mostly takes hits).
Preempted requests wait in one queue and resume oldest first, before any waiting request is admitted: a swapped-out one
when fresh pages for its slots are free (one ``paged_kv_swap`` per step brings back all that resume), straight into the
running set; a recomputed one is admitted like a waiting one and prefilled over all its tokens so far, and the logits
of its last position choose the token the skipped step would have chosen.  Admission and resumption keep enough free
pages for the next step's growth (the next two with chunked prefill, whose steps decode too), so a request is never
prefilled only to be thrown away in the step after.  Beam-search requests keep the whole reservation and are never
victims; neither are admitted prompts, part-way through chunked prefill or not (they hold their prompt's pages and need
none).  Speculative drafts never preempt: they are cut to the pages the request holds plus those the free list can
give.  Every swap runs on the engine's stream and the host never touches the host pool, so stream order is the only
ordering: a swap-out precedes any later write to the pages it frees, and a swap-in the forward that reads its pages.
Works with prefix caching, FP8 pools, speculative decoding, chunked prefill, ``cuda_graphs`` and beam requests.
``preemptions`` counts the preemptions, ``swapped_out_pages`` / ``swapped_in_pages`` the pages swapped, and
``recomputed_tokens`` the positions prefilled again (net of prefix hits; ``cached_prompt_tokens`` counts first
admissions only).  Swap versus recompute is chosen by host room alone, not by cost: see ``docs/KERNELS.md`` for the
measured rates.

Limits: sampled tokens depend on which requests share a step (the random stream is consumed per group; in a verify
step a group takes one uniform number per token row, then one draw per row without the draft, then one per row);
an ``ExpertLayer`` capacity limit counts the tokens of one step, as in ``generate()`` (with prefix caching, cached keys
and values were computed in another step, so with a limit that binds they can differ from a recomputation by more than
rounding).  Tensor-parallel, pipelined and fused NVLink MoE models are refused.
"""
from __future__ import annotations

import bisect
import collections
import itertools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from pipegoose_b200.ops.attention import APPEND_MAX_TOKENS, PAGE_SIZE, fp8_prefill_staging

SPEC_NGRAM_SIZES = (3, 2)                           # trailing n-gram sizes the drafter looks up, longest first
MAX_SPECULATIVE_TOKENS = APPEND_MAX_TOKENS - 1      # drafts per request and step: with the last token, one append
GRAPH_BATCH_SIZES = (1, 2, 4, 8, 16, 32, 64, 128, 256)   # decode batch buckets captured as CUDA graphs (cuda_graphs)
MAX_BEAMS = 8                                       # num_beams of one request: its 2 * num_beams candidates per step


class _NgramIndex:
    """Prompt-lookup drafting for one token list: for every n in ``SPEC_NGRAM_SIZES``, the position of the token that
    followed the most recent occurrence of each n-gram.  ``update`` indexes the tokens appended since its last call, so
    drafting costs O(new tokens) per step, not O(sequence length)."""

    def __init__(self):
        self.index = {n: {} for n in SPEC_NGRAM_SIZES}
        self.seen = 0

    def update(self, tokens: List[int]) -> None:
        for t in range(max(self.seen, 1), len(tokens)):          # token t follows the n-gram tokens[t-n:t]
            for n in SPEC_NGRAM_SIZES:
                if t >= n:
                    self.index[n][tuple(tokens[t - n:t])] = t
        self.seen = len(tokens)

    def draft(self, tokens: List[int], k: int) -> List[int]:
        """Up to ``k`` tokens that followed the most recent earlier occurrence of the trailing n-gram of ``tokens``
        (the longest size that has one), ``[]`` if none.  ``update(tokens)`` comes first."""
        if k <= 0:
            return []
        for n in SPEC_NGRAM_SIZES:
            f = self.index[n].get(tuple(tokens[-n:])) if len(tokens) > n else None
            if f is not None:
                return tokens[f:f + k]
        return []


@dataclass
class _Beam:
    """One running beam of a beam-search request: its tokens (prompt + generated), fp32 running score and pages."""
    tokens: List[int]
    score: float
    pages: List[int]


@dataclass
class _BeamSearch:
    """A beam-search request's state.  ``beams`` are its decode rows in 🤗's order (one row, the prompt, before its
    first beam step); ``finished`` its best finished hypotheses ``(score, generated tokens)``, best first, at most
    ``width``; ``refs`` the request-local references of the pages its beams hold and ``spare`` its reserved pages that
    no beam holds."""
    width: int
    length_penalty: float
    early_stopping: object            # True, False or "never"
    num_return_sequences: int
    beams: List[_Beam] = field(default_factory=list)
    finished: List[Tuple[float, List[int]]] = field(default_factory=list)
    improvable: bool = True           # 🤗's early-stopping heuristic: can a running beam still beat the worst finished
    refs: Dict[int, int] = field(default_factory=dict)
    spare: List[int] = field(default_factory=list)


@dataclass
class _Request:
    rid: int
    tokens: List[int]
    prompt_len: int
    max_new_tokens: int
    sampling: Tuple            # (do_sample, temperature, top_k, top_p): requests with the same tuple are picked together
    eos_token_id: Optional[int]
    pages: List[int] = field(default_factory=list)
    cached: int = 0            # prompt positions served from the prefix cache (a multiple of the page size)
    filled: int = 0            # chunked prefill: prompt positions in the cache so far (at least ``cached``)
    ngrams: Optional[_NgramIndex] = None      # speculative decoding only
    beam: Optional[_BeamSearch] = None        # beam search only
    slots: List[int] = field(default_factory=list)   # preemption: host slots holding its pages while swapped out

    @property
    def pages_needed(self) -> int:
        """Pages reserved at admission: those of the whole sequence; for beam search the prompt's full pages once and
        the rest once per beam."""
        n = -(-(self.prompt_len + self.max_new_tokens) // PAGE_SIZE)
        if self.beam is None:
            return n
        full = self.prompt_len // PAGE_SIZE
        return full + self.beam.width * (n - full)

    def rows(self) -> list:
        """The request's decode rows (objects with ``tokens`` and ``pages``): its beams, or itself."""
        return self.beam.beams if self.beam is not None else [self]


class ContinuousBatcher:
    """Continuous-batching generation for a ``BloomForCausalLM`` / ``GPT2LMHeadModel`` (module docstring).

    ``max_cache_tokens``: KV-cache positions the pools hold (rounded down to whole pages of 64).
    ``max_prefill_tokens``: most prompt tokens packed into one prefill step (tokens served from the prefix cache do
    not count).
    ``generator``: random stream of sampled requests.
    ``prefix_caching``: reuse the pages of earlier prompts that share a prefix (module docstring).
    ``kv_cache_dtype``: ``None`` keeps the pools in the model's dtype, ``torch.float8_e4m3fn`` stores them in FP8 with
    per-position scales (module docstring).
    ``num_speculative_tokens``: most prompt-lookup drafts per request and decode step, 0 .. 7 (module docstring); 0
    turns speculation off.
    ``chunked_prefill``: run prompts in page-aligned chunks of at most ``max_prefill_tokens`` tokens per step, in the
    same steps as the running requests' decode tokens (module docstring); needs ``max_prefill_tokens >= 64`` and no
    speculative decoding.
    ``cuda_graphs``: replay plain decode steps of at most ``GRAPH_BATCH_SIZES[-1]`` requests from CUDA graphs, one per
    batch bucket, captured on first use (module docstring); costs the graphs' memory pool and one capture pause per
    bucket.  Needs a model on the native decode path with ``BloomMLP`` MLPs.
    ``preemption``: give plain requests pages as they grow instead of reserving their whole length at admission, and
    preempt the latest submitted ones when the pool runs out (module docstring).
    ``swap_space_tokens``: positions of the pinned host pool preempted requests are swapped into (rounded down to whole
    pages; 0: every preempted request is recomputed).  Needs ``preemption=True``.

    Beam search: ``submit(..., num_beams=W)`` (module docstring); ``hypotheses`` maps a finished beam request's id to
    its best ``(prompt + tokens, score)``, and ``beam_page_copies`` counts the partial pages its forks copied."""

    def __init__(self, model, max_cache_tokens: int, max_prefill_tokens: int = 8192,
                 generator: Optional[torch.Generator] = None, prefix_caching: bool = False,
                 kv_cache_dtype: Optional[torch.dtype] = None, num_speculative_tokens: int = 0,
                 chunked_prefill: bool = False, cuda_graphs: bool = False, preemption: bool = False,
                 swap_space_tokens: int = 0):
        from pipegoose_b200.models.bloom import BloomMLP, _decodes_incrementally, _native_decode

        if getattr(model, "tp", None) is not None:
            raise ValueError("ContinuousBatcher serves single-GPU models: tensor-parallel models are not supported")
        if getattr(model, "_pg_pipeline_engine", None) is not None:
            raise ValueError("ContinuousBatcher serves single-GPU models: pipelined (PipelineParallel) models are not "
                             "supported")
        blocks = model.transformer.h
        if not all(isinstance(b.mlp, BloomMLP) or _decodes_incrementally(b.mlp) for b in blocks):
            raise ValueError("ContinuousBatcher does not support the fused NVLink MoE layer (its kernels are built "
                             "around token-sharded full sequences); use ExpertLayer MLPs")
        if kv_cache_dtype not in (None, torch.float8_e4m3fn):
            raise ValueError(f"kv_cache_dtype must be None or torch.float8_e4m3fn, got {kv_cache_dtype}")
        if max_prefill_tokens < 1:
            raise ValueError(f"max_prefill_tokens must be at least 1, got {max_prefill_tokens}")
        if not 0 <= num_speculative_tokens <= MAX_SPECULATIVE_TOKENS:
            raise ValueError(f"num_speculative_tokens must be in 0 .. {MAX_SPECULATIVE_TOKENS}, got "
                             f"{num_speculative_tokens}")
        if num_speculative_tokens and kv_cache_dtype is not None:
            raise ValueError("speculative decoding does not support FP8 KV-cache pools")
        if chunked_prefill and max_prefill_tokens < PAGE_SIZE:
            raise ValueError(f"chunked prefill cuts prompts at page boundaries: max_prefill_tokens must be at least "
                             f"{PAGE_SIZE}, got {max_prefill_tokens}")
        if chunked_prefill and num_speculative_tokens:
            raise ValueError("chunked prefill does not support speculative decoding")
        if swap_space_tokens < 0:
            raise ValueError(f"swap_space_tokens must be at least 0, got {swap_space_tokens}")
        if swap_space_tokens and not preemption:
            raise ValueError("swap_space_tokens needs preemption=True: only preempted requests are swapped out")
        w = blocks[0].self_attention.query_key_value.weight
        D = model.config.hidden_size // model.config.n_head
        if cuda_graphs and not all(isinstance(b.mlp, BloomMLP) for b in blocks):
            raise ValueError("cuda_graphs needs BloomMLP MLPs: ExpertLayer routing depends on the data, so its decode "
                             "step cannot be captured")
        if cuda_graphs and not _native_decode(w, D):
            raise ValueError("cuda_graphs needs the native decode path: CUDA bf16 weights and a head size of 64, 80 or "
                             f"128 (got {w.dtype} on {w.device}, head size {D})")
        self.cuda_graphs = bool(cuda_graphs)
        self.graph_decode_steps = 0                               # decode steps served by a graph replay
        self._native = _native_decode(w, D)
        self.vocab_size = model.lm_head.weight.shape[0]
        self.beam_page_copies = 0                                 # partial pages copied by beam forks
        self.hypotheses: Dict[int, List[Tuple[List[int], float]]] = {}   # beam search: rid -> best hypotheses
        self.chunked_prefill = bool(chunked_prefill)
        self.num_speculative_tokens = int(num_speculative_tokens)
        self.speculative_proposed_tokens = 0                      # drafts verified
        self.speculative_accepted_tokens = 0                      # accepted drafts emitted
        cfg = model.config
        self.model = model
        self.max_prefill_tokens = int(max_prefill_tokens)
        self.generator = generator
        self.num_pages = int(max_cache_tokens) // PAGE_SIZE
        if self.num_pages < 1:
            raise ValueError(f"max_cache_tokens = {max_cache_tokens} holds no page of {PAGE_SIZE} positions")
        self.n_positions = cfg.n_positions if getattr(cfg, "position_embedding", "alibi") == "learned" else None
        # with cuda_graphs, one more page (index num_pages) that only the graphs' padding rows write
        shape = (len(blocks), self.num_pages + self.cuda_graphs, cfg.n_head, PAGE_SIZE, D)
        self.k_pools = torch.empty(shape, dtype=kv_cache_dtype or w.dtype, device=w.device)
        self.v_pools = torch.empty(shape, dtype=kv_cache_dtype or w.dtype, device=w.device)
        self.k_scales = self.v_scales = None
        if kv_cache_dtype is not None:
            self.k_scales = torch.empty(shape[:-1], dtype=torch.float32, device=w.device)
            self.v_scales = torch.empty(shape[:-1], dtype=torch.float32, device=w.device)
        self.device = w.device
        self._free = collections.deque(range(self.num_pages))
        self.prefix_caching = bool(prefix_caching)
        self.cached_prompt_tokens = 0                             # prompt tokens served from the prefix cache
        if self.prefix_caching:
            # free pages in the order they were freed, O(1) removal of a revived one
            self._free = collections.OrderedDict.fromkeys(range(self.num_pages))
            self._refs = [0] * self.num_pages
            self._index: Dict[Tuple[int, Tuple[int, ...]], int] = {}    # (parent key id, 64 tokens) -> page
            self._page_key: Dict[int, Tuple[Tuple[int, Tuple[int, ...]], int]] = {}   # page -> (key, key id)
            self._key_ids = itertools.count()
        self._ids = itertools.count()
        self._waiting: collections.deque = collections.deque()    # submitted, no pages yet
        self._admitted: collections.deque = collections.deque()   # pages reserved, prompt not yet (wholly) run
        self._running: List[_Request] = []                        # prompt in the cache, decoding
        self.preemption = bool(preemption)
        self._preempted: List[_Request] = []                      # preempted, oldest first
        self.preemptions = 0                                      # requests preempted (each time counts)
        self.swapped_out_pages = 0
        self.swapped_in_pages = 0
        self.recomputed_tokens = 0                                # positions prefilled again, net of prefix hits
        slots = int(swap_space_tokens) // PAGE_SIZE
        self._host_free = collections.deque(range(slots))
        self.host_kv = self.host_scales = None
        if slots:
            pin = self.device.type == "cuda"
            self.host_kv = torch.empty((slots, shape[0], 2) + shape[2:], dtype=self.k_pools.dtype, pin_memory=pin)
            if self.k_scales is not None:
                self.host_scales = torch.empty((slots, shape[0], 2) + shape[2:-1], dtype=torch.float32, pin_memory=pin)
        if self.cuda_graphs:
            self._init_graphs()

    # ------------------------------------------------------------------ public
    def submit(self, prompt_ids: Sequence[int], max_new_tokens: int, do_sample: bool = False, temperature: float = 1.0,
               top_k: int = 0, top_p: float = 1.0, eos_token_id: Optional[int] = None, num_beams: int = 1,
               length_penalty: float = 1.0, early_stopping=False, num_return_sequences: int = 1) -> int:
        """Queue one request; returns its id.  The arguments mean what they mean in ``generate()`` and 🤗's beam
        search (module docstring).  With ``num_beams > 1`` the request's result is its best hypothesis, and
        ``hypotheses[rid]`` receives its ``num_return_sequences`` best ``(prompt + tokens, score)``, best first, where the
        score is 🤗's ``sequences_scores``; the caller pops those entries."""
        tokens = [int(t) for t in (prompt_ids.reshape(-1).tolist() if torch.is_tensor(prompt_ids) else prompt_ids)]
        if not tokens:
            raise ValueError("empty prompt: a request needs at least one token")
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be at least 1, got {max_new_tokens}")
        if not 1 <= num_beams <= MAX_BEAMS:
            raise ValueError(f"num_beams must be in 1 .. {MAX_BEAMS}, got {num_beams}")
        if not 1 <= num_return_sequences <= num_beams:
            raise ValueError(f"num_return_sequences must be in 1 .. num_beams = {num_beams}, got {num_return_sequences}")
        beam = None
        if num_beams > 1:
            if do_sample:
                raise ValueError("num_beams > 1 does not support do_sample=True (beam sampling)")
            if self.num_speculative_tokens:
                raise ValueError("num_beams > 1 is not supported with speculative decoding (num_speculative_tokens > 0)")
            if early_stopping not in (True, False, "never"):
                raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
            if 2 * num_beams > self.vocab_size:
                raise ValueError(f"num_beams = {num_beams} needs 2 * num_beams candidates per step; the vocabulary has "
                                 f"{self.vocab_size} tokens")
            beam = _BeamSearch(int(num_beams), float(length_penalty), early_stopping, int(num_return_sequences))
        # the last new token is never fed back: positions 0 .. prompt + max_new_tokens - 2 are embedded
        if self.n_positions is not None and len(tokens) + max_new_tokens - 1 > self.n_positions:
            raise ValueError(f"prompt ({len(tokens)}) + max_new_tokens ({max_new_tokens}) - 1 positions exceed the "
                             f"model's n_positions = {self.n_positions}")
        r = _Request(next(self._ids), tokens, len(tokens), int(max_new_tokens),
                     (bool(do_sample), float(temperature), int(top_k), float(top_p)) if do_sample else (False,),
                     eos_token_id, beam=beam)
        if r.pages_needed > self.num_pages:
            what = f" with num_beams {num_beams}" if beam is not None else ""
            raise ValueError(f"the request needs {r.pages_needed} pages of {PAGE_SIZE} positions (prompt {len(tokens)} + "
                             f"max_new_tokens {max_new_tokens}{what}); the pool has {self.num_pages}")
        self._waiting.append(r)
        return r.rid

    def has_work(self) -> bool:
        return bool(self._waiting or self._admitted or self._running or self._preempted)

    def step(self) -> List[Tuple[int, List[int]]]:
        """One prefill, decode or (chunked prefill) mixed step; returns ``(rid, prompt + new tokens)`` of the requests
        that finished."""
        self._admit()
        if self.preemption and (self.chunked_prefill or not self._admitted):
            self._grow()
        spec = self._speculate() if self.num_speculative_tokens and not self._admitted else None
        done = []
        if spec is not None:
            reqs, emitted = spec
        else:
            rows, logits = self._forward()
            if not rows:
                return []
            reqs = [r for r in rows if r.beam is None]              # plain rows come first (_order)
            emitted = [[t] for t in self._select(reqs, logits[:len(reqs)].float())] if reqs else []
            tail = rows[len(reqs):]                                 # beam requests, each with its rows adjacent
            beams = [r for i, r in enumerate(tail) if i == 0 or tail[i - 1] is not r]
            if beams:
                done = self._beam_step(beams, logits[len(reqs):])
        for r, new in zip(reqs, emitted):
            r.tokens += new
            if len(r.tokens) - r.prompt_len == r.max_new_tokens or new[-1] == r.eos_token_id:
                if self.prefix_caching:
                    self._release(r)
                else:
                    self._drop(r.pages)
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
    @staticmethod
    def _order(r: _Request) -> Tuple:
        """Row order of a step: requests that share sampling parameters adjacent, beam-search requests last."""
        return (r.beam is not None, r.sampling)

    def _admit(self) -> None:
        """First come, first served: no request overtakes an earlier one.  With preemption, preempted requests come
        before waiting ones, oldest first; one ``paged_kv_swap`` brings back every swapped-out request that resumes."""
        pairs = []
        for queue in (self._preempted, self._waiting):
            while queue and (self._swap_in(queue[0], pairs) if queue[0].slots else self._take(queue[0])):
                del queue[0]
            if queue:
                break
        if pairs:
            self._swap(pairs, to_host=False)

    def _take(self, r: _Request) -> bool:
        """Admit ``r`` if the free list holds its pages: all it can need (``pages_needed``), or with preemption a plain
        request's pages of ``tokens`` so far, plus ``_headroom``.  Prefix-cache hits take a reference; hit pages on the
        free list count against the free pages they are taken from."""
        hits = self._match(r) if self.prefix_caching else []
        revived = sum(1 for p in hits if self._refs[p] == 0)
        n = (-(-len(r.tokens) // PAGE_SIZE) if self.preemption and r.beam is None else r.pages_needed) - len(hits)
        if n + revived + (self._headroom([r]) if self.preemption else 0) > len(self._free):
            return False
        for p in hits:
            if self._refs[p] == 0:
                del self._free[p]
            self._refs[p] += 1
        r.pages = hits + [self._take_page() for _ in range(n)]
        r.cached, r.filled = len(hits) * PAGE_SIZE, 0
        if not all(0 <= p < self.num_pages for p in r.pages):
            raise RuntimeError(f"page ids {r.pages} outside the pool of {self.num_pages} pages")
        if len(r.tokens) > r.prompt_len:                     # readmitted after a preemption: recomputed
            self.recomputed_tokens += len(r.tokens) - r.cached
        self._admitted.append(r)
        return True

    def _take_page(self) -> int:
        """A page off the free list (with prefix caching the least recently freed one: it loses its index entry, whose
        content is about to change, and takes one reference)."""
        if not self.prefix_caching:
            return self._free.popleft()
        p = self._free.popitem(last=False)[0]
        entry = self._page_key.pop(p, None)
        if entry is not None:
            del self._index[entry[0]]
        self._refs[p] = 1
        return p

    def _drop(self, pages: List[int]) -> None:
        """Return pages to the free list; with prefix caching drop one reference of each, last page first."""
        if not self.prefix_caching:
            self._free.extend(pages)
            return
        for p in reversed(pages):
            self._refs[p] -= 1
            if self._refs[p] == 0:
                self._free[p] = None

    # ------------------------------------------------------------------ preemption
    def _headroom(self, new: List[_Request]) -> int:
        """Pages the free list must keep so that admitting the prompts in ``new``, or resuming its swapped-out requests,
        preempts nothing in the step that follows: those the next write of every running plain request starts (with
        chunked prefill the next two writes: the admitting step decodes too), and those the first decode of every
        admitted plain prompt starts (its pages hold ``len(tokens)`` positions)."""
        ahead, n = int(self.chunked_prefill), 0
        for r in self._running + [x for x in new if x.slots]:
            if r.beam is None:
                n += max(0, (len(r.tokens) - 1 + ahead) // PAGE_SIZE + 1 - len(r.pages or r.slots))
        for r in list(self._admitted) + [x for x in new if not x.slots]:
            n += r.beam is None and len(r.tokens) % PAGE_SIZE == 0
        return n

    def _grow(self) -> None:
        """Before a decode, mixed or verify step: every running plain request whose next write starts a page takes one
        off the free list.  While the free list cannot cover them, the latest submitted running plain request is
        preempted (possibly one of them).  One ``paged_kv_swap``, enqueued before any write to the pages it frees,
        serves the step's swap-outs."""
        plain = sorted((r for r in self._running if r.beam is None), key=lambda r: r.rid)
        short = {r.rid for r in plain if (len(r.tokens) - 1) // PAGE_SIZE >= len(r.pages)}
        pairs = []
        while len(short) > len(self._free):
            r = plain.pop()
            short.discard(r.rid)
            self._preempt(r, pairs)
        if pairs:
            self._swap(pairs, to_host=True)
        for r in plain:
            if r.rid in short:
                r.pages.append(self._take_page())

    def _preempt(self, r: _Request, pairs: List[Tuple[int, int]]) -> None:
        """Take a running request out: swap its pages out if they fit in the free host slots (their ``(page, slot)``
        pairs join ``pairs``), else free them for a recompute (with prefix caching ``_release`` indexes its full pages
        first, so its readmission mostly takes hits).  It waits in the preempted queue."""
        self._running.remove(r)
        self.preemptions += 1
        if len(r.pages) <= len(self._host_free):
            r.slots = [self._host_free.popleft() for _ in r.pages]
            pairs += zip(r.pages, r.slots)
            self.swapped_out_pages += len(r.pages)
            self._drop(r.pages)
        elif self.prefix_caching:
            self._release(r)
        else:
            self._drop(r.pages)
        r.pages = []
        bisect.insort(self._preempted, r, key=lambda x: x.rid)

    def _swap_in(self, r: _Request, pairs: List[Tuple[int, int]]) -> bool:
        """Resume a swapped-out request if fresh pages for its slots, plus ``_headroom``, are free: its ``(page, slot)``
        pairs join ``pairs`` and it rejoins the running set."""
        if len(r.slots) + self._headroom([r]) > len(self._free):
            return False
        r.pages = [self._take_page() for _ in r.slots]
        pairs += zip(r.pages, r.slots)
        self._host_free.extend(r.slots)
        self.swapped_in_pages += len(r.slots)
        r.slots = []
        self._running.append(r)
        return True

    def _swap(self, pairs: List[Tuple[int, int]], to_host: bool) -> None:
        from pipegoose_b200.ops.attention import paged_kv_swap

        paged_kv_swap(pairs, self.k_pools, self.v_pools, self.k_scales, self.v_scales, self.host_kv, self.host_scales,
                      to_host)

    # ------------------------------------------------------------------ prefix cache
    def _match(self, r: _Request) -> List[int]:
        """Indexed pages holding the prompt's leading full pages, at most ``(prompt - 1) // 64``."""
        hits, parent = [], -1
        for k in range((len(r.tokens) - 1) // PAGE_SIZE):
            page = self._index.get((parent, tuple(r.tokens[k * PAGE_SIZE:(k + 1) * PAGE_SIZE])))
            if page is None:
                break
            hits.append(page)
            parent = self._page_key[page][1]
        return hits

    def _register(self, r: _Request, filled: int) -> None:
        """Index the request's full pages among positions ``0 .. filled-1`` (all written to the pools).  A key that is
        already indexed keeps its first page; the chain continues from that page's key id."""
        parent = -1
        for k in range(filled // PAGE_SIZE):
            page = r.pages[k]
            entry = self._page_key.get(page)
            if entry is None:
                key = (parent, tuple(r.tokens[k * PAGE_SIZE:(k + 1) * PAGE_SIZE]))
                first = self._index.get(key)
                if first is not None:
                    entry = self._page_key[first]
                else:
                    entry = (key, next(self._key_ids))
                    self._index[key] = page
                    self._page_key[page] = entry
            parent = entry[1]

    def _release(self, r: _Request) -> None:
        """A finished request: index the pages its generated tokens filled (positions up to ``len(tokens) - 2`` are in
        the cache; a beam-search request indexes its prompt only), then drop its references, last page first."""
        self._register(r, r.prompt_len if r.beam is not None else len(r.tokens) - 1)
        self._drop(r.pages)

    def _upload(self, rows: List[List[int]]) -> List[torch.Tensor]:
        """Host int lists -> int32 device tensors, in one copy."""
        flat = torch.tensor(list(itertools.chain.from_iterable(rows)), dtype=torch.int32).to(self.device)
        return list(flat.split([len(r) for r in rows]))

    def _forward(self) -> Tuple[List[_Request], torch.Tensor]:
        """The owner of every row this step serves (a beam-search request owns one row per beam), in ``_order``, and
        the rows' next-token logits ``[len(rows), V]`` in the model's dtype."""
        if self._admitted and self.chunked_prefill:
            return self._mixed()
        if self._admitted:                                      # prefill the oldest admitted prompts
            reqs, n = [], 0
            while self._admitted and (not reqs or n + len(self._admitted[0].tokens) - self._admitted[0].cached
                                      <= self.max_prefill_tokens):
                reqs.append(self._admitted.popleft())
                n += len(reqs[-1].tokens) - reqs[-1].cached
            reqs.sort(key=self._order)
            if self.prefix_caching:
                logits = self._prefill_cached(reqs) if any(r.cached for r in reqs) else self._prefill(reqs)
                for r in reqs:
                    if len(r.tokens) == r.prompt_len:            # a first admission, not a recompute
                        self.cached_prompt_tokens += r.cached
                    self._register(r, len(r.tokens))
                return reqs, logits
            return reqs, self._prefill(reqs)
        reqs = sorted(self._running, key=self._order)
        self._running = []
        if not reqs:
            return [], None
        owners = [r for r in reqs for _ in r.rows()]
        rows = [b for r in reqs for b in r.rows()]
        if self.cuda_graphs and len(rows) <= self._graph_sizes[-1]:
            return owners, self._graph_decode(rows)
        width = max(len(b.pages) for b in rows)
        table = [p for b in rows for p in b.pages + [0] * (width - len(b.pages))]
        pos = [len(b.tokens) - 1 for b in rows]
        ids, positions, table = self._upload([[b.tokens[-1] for b in rows], pos, table])
        logits = self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, table=table.view(len(rows), width),
                                          max_pos=max(pos), k_scales=self.k_scales, v_scales=self.v_scales)
        return owners, logits

    def _prefill(self, reqs: List[_Request]) -> torch.Tensor:
        """Whole prompts packed into one row through the document-masked flash kernel."""
        ids, positions, seg, slot, last, o = [], [], [], [], [], 0
        for r in reqs:
            P = len(r.tokens)
            ids += r.tokens
            positions += range(P)
            seg += [o] * P
            slot += [r.pages[p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE for p in range(P)]
            o += P
            last.append(o - 1)
        ids, positions, seg, slot, last = self._upload([ids, positions, seg, slot, last])
        return self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, seg_start=seg, slot=slot,
                                        last=last, k_scales=self.k_scales, v_scales=self.v_scales)

    def _prefill_cached(self, reqs: List[_Request]) -> torch.Tensor:
        """The prompts' uncached suffixes, packed back to back, through the paged prefill kernel over the pools (over a
        bf16 staging pool with FP8 pools: its plan goes in the step's upload)."""
        ids, positions, slot, last, cu, start, o = [], [], [], [], [0], [], 0
        width = max(len(r.pages) for r in reqs)
        table = []
        for r in reqs:
            P, st = len(r.tokens), r.cached
            ids += r.tokens[st:P]
            positions += range(st, P)
            slot += [r.pages[p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE for p in range(st, P)]
            o += P - st
            last.append(o - 1)
            cu.append(o)
            start.append(st)
            table += r.pages + [0] * (width - len(r.pages))
        max_len = max(len(r.tokens) - r.cached for r in reqs)
        n, plan = self._staging([r.pages for r in reqs], [r.cached for r in reqs], [len(r.tokens) for r in reqs])
        up = self._upload([ids, positions, slot, last, cu, start, table] + plan)
        ids, positions, slot, last, cu, start, table = up[:7]
        stage = (n, up[7], up[8], up[9], up[10].view(len(reqs), -1)) if plan else None
        return self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, slot=slot, last=last,
                                        table=table.view(len(reqs), width), cu_seqlens=cu, start=start,
                                        max_len=max_len, k_scales=self.k_scales, v_scales=self.v_scales, stage=stage)

    def _staging(self, pages: List[List[int]], starts: List[int], ends: List[int]) -> Tuple[int, List[List[int]]]:
        """FP8 pools: the staging plan (:func:`fp8_prefill_staging`) of a prefill whose sequences have ``starts``
        positions in the pools and ``ends`` in all, as its pool size and host rows for the step's upload; ``(0, [])``
        with other pools."""
        if self.k_scales is None:
            return 0, []
        n, src, dst, slot, table = fp8_prefill_staging(pages, starts, ends)
        return n, [src, dst, slot, [p for row in table for p in row]]

    def _chunks(self) -> List[Tuple[_Request, int, int]]:
        """The step's prompt chunks ``(request, first position, end)``, first come, first served, at most
        ``max_prefill_tokens`` tokens in all.  A chunk that does not end its prompt ends on a page boundary, and no
        later request gets a chunk in that step."""
        chunks, n = [], 0
        for r in self._admitted:
            s = max(r.filled, r.cached)
            room = self.max_prefill_tokens - n
            P = len(r.tokens)
            e = P if P - s <= room else (s + room) // PAGE_SIZE * PAGE_SIZE
            if e > s:
                chunks.append((r, s, e))
                n += e - s
            if e < P:
                break
        return chunks

    def _mixed(self) -> Tuple[List[_Request], torch.Tensor]:
        """Chunked prefill: one decode token of every running request's rows (its beams, for beam search), then the
        step's prompt chunks, through one forward.  Requests whose prompt completes choose their first token (make
        their first beam step) from their last prompt row in this step; the others stay admitted."""
        owners = [r for r in self._running for _ in r.rows()]
        dec = [b for r in self._running for b in r.rows()]
        self._running = []
        chunks = self._chunks()
        width = max(len(r.pages) for r in dec + [c[0] for c in chunks])
        ids = [r.tokens[-1] for r in dec]
        positions = [len(r.tokens) - 1 for r in dec]
        table = [p for r in dec + [c[0] for c in chunks] for p in r.pages + [0] * (width - len(r.pages))]
        slot, cu, start, done, rows = [], [0], [], [], list(range(len(dec)))
        for r, s, e in chunks:
            ids += r.tokens[s:e]
            positions += range(s, e)
            slot += [r.pages[p // PAGE_SIZE] * PAGE_SIZE + p % PAGE_SIZE for p in range(s, e)]
            cu.append(cu[-1] + e - s)
            start.append(s)
            r.filled = e
            if e == len(r.tokens):
                done.append(r)
                rows.append(len(dec) + cu[-1] - 1)
        for r in done:                                          # the oldest admitted requests
            self._admitted.popleft()
            if self.prefix_caching:
                if len(r.tokens) == r.prompt_len:                # a first admission, not a recompute
                    self.cached_prompt_tokens += r.cached
                self._register(r, len(r.tokens))
        reqs = owners + done
        order = sorted(range(len(reqs)), key=lambda i: self._order(reqs[i]))  # stable: groups, each beam's rows, adjacent
        last = [rows[i] for i in order]
        n, plan = self._staging([r.pages for r, _, _ in chunks], start, [e for _, _, e in chunks])
        up = self._upload([ids, positions, table, slot, cu, start, last] + plan)
        ids, positions, table, slot, cu, start, last = up[:7]
        stage = (n, up[7], up[8], up[9], up[10].view(len(chunks), -1)) if plan else None
        logits = self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, slot=slot, last=last,
                                          table=table.view(-1, width), max_pos=max([0] + [len(r.tokens) - 1 for r in dec]),
                                          cu_seqlens=cu, start=start, max_len=max(e - s for _, s, e in chunks),
                                          k_scales=self.k_scales, v_scales=self.v_scales, stage=stage,
                                          n_dec=len(dec))
        return [reqs[i] for i in order], logits

    # ------------------------------------------------------------------ CUDA graphs
    def _init_graphs(self) -> None:
        """The decode graphs' static inputs: one int32 device buffer and its pinned host mirror.  Bucket n uses the
        prefix ``ids [n] | positions [n] | table [n, W]``, W the most pages one request can reserve."""
        self._graph_sizes = tuple(sorted(GRAPH_BATCH_SIZES))
        self._graph_width = self.num_pages
        if self.n_positions is not None:            # a request holds at most n_positions + 1 positions (submit)
            self._graph_width = min(self.num_pages, -(-(self.n_positions + 1) // PAGE_SIZE))
        size = self._graph_sizes[-1] * (2 + self._graph_width)
        self._graph_in = torch.zeros(size, dtype=torch.int32, device=self.device)
        self._graph_host = torch.zeros(size, dtype=torch.int32).pin_memory()
        self._graphs: Dict[int, Tuple] = {}                         # bucket -> (graph, static logits, decode tickets)
        self._graph_pool = torch.cuda.graph_pool_handle()
        self._graph_stream = torch.cuda.Stream(self.device)

    def _graph_inputs(self, n: int, ids: List[int], positions: List[int],
                      pages: List[List[int]]) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Fill bucket ``n``'s static inputs, in one host-to-device copy: the ``len(ids)`` rows given, then padding rows
        (token 0 at position 0, a table row of the scratch page ``num_pages``); returns the device views ``ids [n]``,
        ``positions [n]`` and ``table [n, W]``.  Table entries behind a row's pages keep older values: the kernel reads
        only the pages of positions ``0 .. positions[b]``.

        Invariant: padding rows write their key and value into slot 0 of the scratch page and read only that key, from
        their own qkv row (the decode kernel takes the key at ``positions[b]`` from qkv), so no real row ever reads the
        scratch page and the padding rows' concurrent writes to it are harmless."""
        W, B, scratch = self._graph_width, len(ids), self.num_pages
        host = self._graph_host[:n * (2 + W)]
        host[:2 * n] = torch.tensor(ids + [0] * (n - B) + positions + [0] * (n - B), dtype=torch.int32)
        table = host[2 * n:].view(n, W)
        if B:
            w = max(len(p) for p in pages)
            table[:B, :w] = torch.tensor([p + [scratch] * (w - len(p)) for p in pages], dtype=torch.int32)
        table[B:] = scratch
        dev = self._graph_in[:host.numel()]
        dev.copy_(host, non_blocking=True)
        return dev[:n], dev[n:2 * n], dev[2 * n:].view(n, W)

    def _graph_call(self, ids: torch.Tensor, positions: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
        """The decode forward a graph holds, on static inputs: logits ``[n, V]`` in the model's dtype."""
        return self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, table=table,
                                        max_pos=self._graph_width * PAGE_SIZE - 1, k_scales=self.k_scales,
                                        v_scales=self.v_scales)

    def _graph(self, n: int) -> Tuple:
        """Bucket ``n``'s ``(graph, static logits [n, V], decode tickets)``, captured on first use.  Warm-up and capture
        run on all-padding inputs, so they write only the scratch page while the pools hold live requests."""
        from pipegoose_b200.ops.attention import _decode_ticket

        if n in self._graphs:
            return self._graphs[n]
        inputs = self._graph_inputs(n, [], [], [])
        s = self._graph_stream
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            # one eager call first: the decode-ticket array (zero-filled), the ALiBi slope caches and cuBLAS's handle
            # and workspace are made on first use, and a capture would only record their initialisation
            self._graph_call(*inputs)
        s.synchronize()                                   # the host mirror is refilled before the replay
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=self._graph_pool, stream=s):
            logits = self._graph_call(*inputs)
        # the graph keeps using the ticket array it captured: hold it, since a larger eager step replaces the cached one
        self._graphs[n] = (graph, logits, _decode_ticket(0, self.device))
        return self._graphs[n]

    def _graph_decode(self, reqs: list) -> torch.Tensor:
        """The plain decode step by graph replay: logits ``[len(reqs), V]``, the first rows of the bucket's, for decode
        rows ``reqs`` (requests or beams: ``tokens`` and ``pages``)."""
        n = next(s for s in self._graph_sizes if s >= len(reqs))
        graph, logits, _ = self._graph(n)
        self._graph_inputs(n, [r.tokens[-1] for r in reqs], [len(r.tokens) - 1 for r in reqs], [r.pages for r in reqs])
        graph.replay()
        self.graph_decode_steps += 1
        return logits[:len(reqs)]

    def _select(self, reqs: List[_Request], logits: torch.Tensor) -> List[int]:
        """Next token of every request (``reqs`` grouped by sampling parameters), one device-to-host transfer."""
        picks, i = [], 0
        for key, group in itertools.groupby(reqs, key=lambda r: r.sampling):
            n = len(list(group))
            do_sample, temperature, top_k, top_p = key if key[0] else (False, 1.0, 0, 1.0)
            picks.append(self.model._select_token(logits[i:i + n], do_sample, temperature, top_k, top_p, self.generator))
            i += n
        return torch.cat(picks).tolist()

    # ------------------------------------------------------------------ beam search
    def _beam_step(self, reqs: List[_Request], logits: torch.Tensor) -> List[Tuple[int, List[int]]]:
        """One beam step of every beam-search request in ``reqs`` from its rows of ``logits`` (model dtype, each
        request's rows adjacent, in ``reqs`` order), as 🤗's ``_beam_search`` makes it: the 2W best candidates
        (``beam_topk``), finished hypotheses, the next W beams and the stopping test.  Running requests fork their
        beams (``_fork``); one ``paged_kv_copy`` serves every copy of the step.  Returns ``(rid, prompt + best
        hypothesis)`` of the requests that finished, whose pages are released."""
        from pipegoose_b200.ops.attention import paged_kv_copy
        from pipegoose_b200.ops.kernels import beam_topk, beam_topk_reference

        for r in reqs:
            if not r.beam.beams:                     # first step: the prompt's row, score 0
                prompt = -(-r.prompt_len // PAGE_SIZE)
                r.beam.beams = [_Beam(list(r.tokens), 0.0, r.pages[:prompt])]
                r.beam.refs = dict.fromkeys(r.pages[:prompt], 1)
                r.beam.spare = list(r.pages[prompt:])
        cu, scores = [0], []
        for r in reqs:
            cu.append(cu[-1] + len(r.beam.beams))
            scores += [b.score for b in r.beam.beams]
        k = 2 * max(r.beam.width for r in reqs)
        topk = beam_topk if self._native else beam_topk_reference
        sc, tok, row, _ = topk(logits, torch.tensor(scores, dtype=torch.float32), cu, k)
        host = torch.cat([sc.view(torch.int32), tok.int(), row.int()]).cpu()        # one device-to-host transfer
        sc, tok, row = host[:len(reqs)].view(torch.float32).tolist(), host[len(reqs):2 * len(reqs)].tolist(), \
            host[2 * len(reqs):].tolist()
        done, copies = [], []
        for i, r in enumerate(reqs):
            b = r.beam
            W = b.width
            cands = [(sc[i][j], tok[i][j], row[i][j] - cu[i]) for j in range(2 * W)]
            gen = len(b.beams[0].tokens) - r.prompt_len                  # tokens generated before this step
            hit = [t == r.eos_token_id or gen + 1 >= r.max_new_tokens for _, t, _ in cands]
            # finished hypotheses: candidates among the top W that end here, length-penalised (🤗's fp32 arithmetic)
            if b.improvable and not (len(b.finished) == W and b.early_stopping is True):
                div = np.float32((gen + 1) ** b.length_penalty)
                new = [(float(np.float32(s) / div), b.beams[p].tokens[r.prompt_len:] + [t])
                       for (s, t, p), h in zip(cands[:W], hit[:W]) if h]
                b.finished = sorted(b.finished + new, key=lambda f: -f[0])[:W]        # stable
            running = [c for c, h in zip(cands, hit) if not h][:W]
            if b.improvable and len(b.finished) == W and running:
                length = r.max_new_tokens if b.early_stopping == "never" and b.length_penalty > 0 else gen + 1
                best = np.float32(running[0][0]) / np.float32(length ** b.length_penalty)
                b.improvable = bool(best > np.float32(b.finished[-1][0]))
            if all(hit) or not b.improvable or (len(b.finished) == W and b.early_stopping is True):
                r.tokens = r.tokens[:r.prompt_len] + b.finished[0][1]
                self.hypotheses[r.rid] = [(r.tokens[:r.prompt_len] + g, s) for s, g in
                                          b.finished[:b.num_return_sequences]]
                if self.prefix_caching:
                    self._release(r)
                else:
                    self._drop(r.pages)
                r.pages, r.beam.beams = [], []
                done.append((r.rid, r.tokens))
                continue
            copies += self._fork(r, running)
            self._running.append(r)
        if copies:
            paged_kv_copy(copies, self.k_pools, self.v_pools, self.k_scales, self.v_scales)
            self.beam_page_copies += len(copies)
        return done

    def _fork(self, r: _Request, running: List[Tuple[float, int, int]]) -> List[Tuple[int, int, int]]:
        """The request's next beams ``running`` (score, token, parent index), in 🤗's order, each taking its parent's
        page list; returns the ``(src, dst, count)`` copies this makes.  Pages are reference-counted within the
        request: the new beams' references are taken before the old beams' are dropped, and a page no beam holds
        returns to the request's spare pages.  Copy-on-write: the page holding a beam's next write position
        ``len(tokens) - 1`` must be that beam's alone.  The first of its holders in 🤗's order keeps it; every other gets
        a spare page with the leading ``pos % 64`` slots copied.  At ``pos % 64 == 0`` the write starts a fresh page."""
        b = r.beam
        beams = [_Beam(b.beams[p].tokens + [t], s, list(b.beams[p].pages)) for s, t, p in running]
        for x in beams:
            for p in x.pages:
                b.refs[p] += 1
        for x in b.beams:
            for p in x.pages:
                b.refs[p] -= 1
                if b.refs[p] == 0:
                    del b.refs[p]
                    b.spare.append(p)
        copies, kept = [], set()
        for x in beams:
            k, off = divmod(len(x.tokens) - 1, PAGE_SIZE)
            if off == 0:
                x.pages.append(self._spare_page(r))
                continue
            page = x.pages[k]
            if page not in kept:
                kept.add(page)
                continue
            fresh = self._spare_page(r)
            b.refs[page] -= 1
            x.pages[k] = fresh
            copies.append((page, fresh, off))
        b.beams = beams
        return copies

    def _spare_page(self, r: _Request) -> int:
        """One of the request's spare pages, referenced once by the beam that takes it."""
        if not r.beam.spare:
            raise RuntimeError(f"beam-search request {r.rid} needs more than the {len(r.pages)} pages it reserved")
        p = r.beam.spare.pop()
        r.beam.refs[p] = 1
        return p

    # ------------------------------------------------------------------ speculative decoding
    def _draft(self, r: _Request) -> List[int]:
        """Prompt-lookup drafts of a running request, at most ``max_new_tokens - generated - 1`` of them so that every
        position the step writes lies in the pages reserved at admission (with preemption ``_speculate`` cuts them to
        the pages the request holds and the free list can give)."""
        if r.ngrams is None:
            r.ngrams = _NgramIndex()
        r.ngrams.update(r.tokens)
        budget = r.max_new_tokens - (len(r.tokens) - r.prompt_len) - 1
        return r.ngrams.draft(r.tokens, min(self.num_speculative_tokens, budget))

    def _speculate(self) -> Optional[Tuple[List[_Request], List[List[int]]]]:
        """A verify step: every running request appends its last token and its drafts through the paged append
        kernel, and keeps the drafts verification accepts plus one more token.  None when no request has a draft: the
        step is then the plain decode step."""
        reqs = sorted(self._running, key=lambda r: r.sampling)
        drafts = [self._draft(r) for r in reqs]
        if self.preemption:                          # drafts take free pages but never preempt
            for i, r in enumerate(reqs):
                drafts[i] = d = drafts[i][:max(0, (len(r.pages) + len(self._free)) * PAGE_SIZE - len(r.tokens))]
                while len(r.pages) * PAGE_SIZE < len(r.tokens) + len(d):
                    r.pages.append(self._take_page())
        if not any(drafts):
            return None
        self._running = []
        width = max(len(r.pages) for r in reqs)
        ids, positions, cu, table = [], [], [0], []
        for r, d in zip(reqs, drafts):
            p = len(r.tokens) - 1
            ids += [r.tokens[-1]] + d
            positions += range(p, p + 1 + len(d))
            cu.append(len(ids))
            table += r.pages + [0] * (width - len(r.pages))
        ids, positions, cu, table = self._upload([ids, positions, cu, table])
        logits = self.model._paged_logits(ids, positions, self.k_pools, self.v_pools, table=table.view(len(reqs), width),
                                          max_pos=max(len(r.tokens) - 1 + len(d) for r, d in zip(reqs, drafts)),
                                          cu_seqlens=cu, max_len=1 + max(len(d) for d in drafts))
        emitted = verify_drafts([r.sampling for r in reqs], drafts, ids, logits.float(), self.generator)
        for r, d, new in zip(reqs, drafts, emitted):
            accepted = len(new) - 1                      # the drafts come first, then one token of the verifier
            room = r.max_new_tokens - (len(r.tokens) - r.prompt_len)
            new[:] = new[:room]
            if r.eos_token_id in new:
                del new[new.index(r.eos_token_id) + 1:]
            self.speculative_proposed_tokens += len(d)
            self.speculative_accepted_tokens += min(accepted, len(new))     # accepted drafts that are emitted
        return reqs, emitted


def verify_drafts(samplings: List[Tuple], drafts: List[List[int]], ids: torch.Tensor, logits: torch.Tensor,
                  generator: Optional[torch.Generator] = None) -> List[List[int]]:
    """The tokens each request of a verify step emits: its accepted drafts, then one more token, chosen at the first
    rejected draft or after the last one.  ``samplings`` are the requests' sampling tuples (equal ones adjacent);
    ``ids`` / ``logits [N, V]`` are the step's token rows, each request's last token and then its ``drafts``, so row
    i of a request scores the draft ``ids[i + 1]``.

    Greedy requests accept a draft while it equals the arg-max, and emit the arg-max where they stop.  Sampled
    requests accept draft x at row i with probability p_i(x), where p_i is the filtered distribution
    (``filter_logits``) non-speculative sampling draws from; on a rejection they draw from p_i without x,
    renormalised, and after the last draft from p_i.  The drafts are deterministic, so the emitted tokens follow the
    distribution of non-speculative sampling.  Per sampled group, the random stream gives one uniform number per row,
    then one draw per row from the distribution without the draft, then one per row from p_i.  One device-to-host
    transfer serves all groups."""
    from pipegoose_b200.models.bloom import filter_logits

    target = torch.cat([ids[1:], ids[-1:]]).long().view(-1, 1)
    groups = [(key, len(list(g))) for key, g in itertools.groupby(samplings)]
    outs, row, r0 = [], 0, 0
    for key, n in groups:
        m = sum(1 + len(d) for d in drafts[r0:r0 + n])
        lg, t = logits[row:row + m], target[row:row + m]
        if not key[0]:
            a = lg.argmax(-1)
            outs.append(torch.stack([(a == t.view(-1)).long(), a, a], 1))
        else:
            p = filter_logits(lg, *key[1:]).softmax(-1)
            accept = torch.rand(m, device=p.device, generator=generator) < p.gather(-1, t).view(-1)
            rest = p.scatter(-1, t, 0.0)
            rest = torch.where(rest.sum(-1, keepdim=True) > 0, rest, p)      # p(x) = 1: x is never rejected
            outs.append(torch.stack([accept.long(), torch.multinomial(rest, 1, generator=generator).view(-1),
                                     torch.multinomial(p, 1, generator=generator).view(-1)], 1))
        row += m
        r0 += n
    verdicts = torch.cat(outs).tolist()          # per row: (draft accepted, token if not, token after the last draft)
    emitted, row = [], 0
    for d in drafts:
        new = []
        for j, x in enumerate(d):
            ok, other, _ = verdicts[row + j]
            new.append(x if ok else other)
            if not ok:
                break
        else:
            new.append(verdicts[row + len(d)][2])
        emitted.append(new)
        row += 1 + len(d)
    return emitted
