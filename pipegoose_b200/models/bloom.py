"""H100-native Bloom (``BloomForCausalLM``) with the same module tree and parameter names as
🤗 transformers' Bloom, so HF state dicts load unchanged and the name-based parallel mappings
(reference nn/tensor_parallel/parallel_mapping.py:4-52) apply to both.

The forward is built from the four fused sub-layer functions in ``pipegoose_b200.ops.functional``;
activations are 2-D ``[tokens, hidden]`` bf16 tensors (token-sharded under tensor parallelism),
attention is the flash ALiBi kernel, the lm_head is fused with a vocab-parallel cross entropy
(no ``[tokens, vocab]`` fp32 tensor, no all-gather of logits).

Dropout: Bloom's ``hidden_dropout`` / ``attention_dropout`` default to 0.0, which is what the fully fused sub-layers
implement.  ``hidden_dropout > 0`` (🤗 Bloom's ``dropout_add`` after the attention projection and after the MLP) is
supported in training through a composed path: the same kernels with the residual add taken out of the GEMM epilogue
and ``dropout(.) + residual`` applied between them.  ``attention_dropout > 0`` (on the attention probabilities) takes
the same composed path with the flash kernel replaced by ``ops.attention.alibi_attention_with_dropout`` (probabilities
materialised a head group at a time).  Both only act in ``train()`` mode; ``eval()`` always runs the fused sub-layers.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from pipegoose_b200.ops import functional as PF
from pipegoose_b200.ops import kernels as K


@dataclass
class BloomConfig:
    """Subset of transformers.BloomConfig that defines the architecture."""

    vocab_size: int = 250880
    hidden_size: int = 64
    n_layer: int = 2
    n_head: int = 8
    layer_norm_epsilon: float = 1e-5
    initializer_range: float = 0.02
    hidden_dropout: float = 0.0
    attention_dropout: float = 0.0
    apply_residual_connection_post_layernorm: bool = False
    tie_word_embeddings: bool = True
    # "block": keep only each block's input and recompute its activations during backward (~1/3 more forward FLOPs
    # for ~n_layer x fewer saved activations); "none": save everything (default, fastest)
    recompute: str = "none"
    # architecture switches used by the other model families built from the same blocks (models/gpt2.py):
    # "alibi" (Bloom) or "learned" absolute position embeddings; LayerNorm right after the token embedding or not
    position_embedding: str = "alibi"
    n_positions: int = 0
    embedding_layernorm: bool = True
    # FP8 training of the blocks' four linear layers (qkv, dense, fc1, fc2; forward, dgrad, wgrad) on the FP8 wgmma GEMM:
    # e4m3 activations and weights, e5m2 gradients, one scale per tensor taken from the tensor being cast (no amax
    # history: checkpoints, resume and recompute are unchanged).  LayerNorm, attention, GELU, the residual stream,
    # embeddings, the lm_head and the optimizer (fp32 master weights and main grads) stay as they are.  Needs the native
    # path (CUDA bf16 model), token counts / widths that are multiples of 16 and a head size the flash kernel runs
    # (D <= 128, a multiple of 8; D = 80 runs zero-padded as in bf16); refused (ValueError) under tensor
    # parallelism, with dropout in training and with a replaced MLP (ExpertLayer / fused MoE).  Data parallelism, ZeRO-1,
    # pipeline stages and recompute="block" take it but have not been run with it on several GPUs.  KV-cached
    # generate() and ContinuousBatcher keep using the bf16 weights.
    fp8: bool = False

    @classmethod
    def from_hf(cls, hf_config) -> "BloomConfig":
        return cls(
            vocab_size=hf_config.vocab_size,
            hidden_size=hf_config.hidden_size,
            n_layer=hf_config.n_layer,
            n_head=hf_config.n_head,
            layer_norm_epsilon=hf_config.layer_norm_epsilon,
            initializer_range=hf_config.initializer_range,
            hidden_dropout=hf_config.hidden_dropout,
            attention_dropout=hf_config.attention_dropout,
            apply_residual_connection_post_layernorm=hf_config.apply_residual_connection_post_layernorm,
        )

    def to_hf(self):
        """The 🤗 ``transformers.BloomConfig`` of this architecture."""
        from transformers import BloomConfig as HFConfig

        return HFConfig(vocab_size=self.vocab_size, hidden_size=self.hidden_size, n_layer=self.n_layer, n_head=self.n_head,
                        layer_norm_epsilon=self.layer_norm_epsilon, initializer_range=self.initializer_range,
                        hidden_dropout=self.hidden_dropout, attention_dropout=self.attention_dropout,
                        apply_residual_connection_post_layernorm=self.apply_residual_connection_post_layernorm,
                        tie_word_embeddings=True)

    @classmethod
    def bloom_tiny(cls):
        """A toy size for CPU smoke runs of the examples."""
        return cls(vocab_size=1024, hidden_size=128, n_layer=4, n_head=8)

    @classmethod
    def bloom_560m(cls):
        return cls(hidden_size=1024, n_layer=24, n_head=16)

    @classmethod
    def bloom_1b7(cls):
        return cls(hidden_size=2048, n_layer=24, n_head=16)

    @classmethod
    def bloom_3b(cls):
        return cls(hidden_size=2560, n_layer=30, n_head=32)

    @classmethod
    def bloom_7b1(cls):
        return cls(hidden_size=4096, n_layer=30, n_head=32)


@dataclass
class CausalLMOutput:
    loss: Optional[torch.Tensor] = None
    logits: Optional[torch.Tensor] = None

    def __getitem__(self, i):
        return (self.loss, self.logits)[i]


class BloomAttention(nn.Module):
    def __init__(self, config: BloomConfig):
        super().__init__()
        h = config.hidden_size
        self.hidden_size = h
        self.num_heads = config.n_head
        self.head_dim = h // config.n_head
        self.query_key_value = nn.Linear(h, 3 * h, bias=True)
        self.dense = nn.Linear(h, h, bias=True)
        self.use_alibi = getattr(config, "position_embedding", "alibi") == "alibi"
        self._slopes_cache = {}


class BloomMLP(nn.Module):
    def __init__(self, config: BloomConfig):
        super().__init__()
        h = config.hidden_size
        self.dense_h_to_4h = nn.Linear(h, 4 * h)
        self.dense_4h_to_h = nn.Linear(4 * h, h)

    def forward(self, hidden_states: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        """HF-compatible signature ``mlp(layernorm_output, residual)`` (used by the MoE wrapper)."""
        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        y = PF.mlp_residual(x, self.dense_h_to_4h.weight, self.dense_h_to_4h.bias,
                            self.dense_4h_to_h.weight, self.dense_4h_to_h.bias, residual.reshape(-1, shape[-1]))
        return y.view(shape)


class BloomBlock(nn.Module):
    def __init__(self, config: BloomConfig):
        super().__init__()
        h = config.hidden_size
        self.eps = config.layer_norm_epsilon
        self.input_layernorm = nn.LayerNorm(h, eps=self.eps)
        self.self_attention = BloomAttention(config)
        self.post_attention_layernorm = nn.LayerNorm(h, eps=self.eps)
        self.mlp = BloomMLP(config)
        self.hidden_dropout = float(getattr(config, "hidden_dropout", 0.0))
        self.fp8 = bool(getattr(config, "fp8", False))
        self.tp = None  # set by TensorParallel (sequence-parallel communicator)

    def _check_fp8(self) -> None:
        """``fp8=True`` cases without an FP8 path: refused rather than run in bf16."""
        if self.tp is not None:
            raise ValueError("fp8=True does not support tensor parallelism: the fused all-gather / reduce-scatter GEMMs "
                             "are bf16")
        if self.training and (getattr(self, "hidden_dropout", 0.0) > 0.0 or getattr(self, "attention_dropout", 0.0) > 0.0):
            raise ValueError("fp8=True does not support training with dropout > 0 (hidden_dropout / attention_dropout)")
        if not isinstance(self.mlp, BloomMLP):
            raise ValueError(f"fp8=True needs the dense BloomMLP; this block's MLP was replaced by "
                             f"{type(self.mlp).__name__} (ExpertLayer / fused MoE), which has no FP8 path")

    def _forward_with_dropout(self, x: torch.Tensor, batch: int, seq: int,
                              seg_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``hidden_dropout > 0`` or ``attention_dropout > 0`` in training: ``x + dropout(dense(attention))`` and
        ``x + dropout(mlp)`` — the kernels of the fused path with the residual add applied after the dropout instead of
        in the GEMM epilogue; attention probabilities are dropped in ``alibi_attention_with_dropout``."""
        import torch.nn.functional as F

        from pipegoose_b200.ops.attention import alibi_attention

        attn, tp, p = self.self_attention, self.tp, self.hidden_dropout
        n_head_local = attn.query_key_value.weight.shape[0] // (3 * attn.head_dim)
        zero = torch.zeros_like(x)
        qkv = PF.layernorm_linear(x, self.input_layernorm.weight, self.input_layernorm.bias,
                                  attn.query_key_value.weight, attn.query_key_value.bias, self.eps, tp)
        att = alibi_attention(qkv, attn.alibi_slopes_local(n_head_local), batch, seq, n_head_local, attn.head_dim,
                              dropout_p=getattr(self, "attention_dropout", 0.0), seg_start=seg_start)
        x = x + F.dropout(PF.linear_residual(att, attn.dense.weight, attn.dense.bias, zero, tp), p, True)
        mlp = self.mlp
        if isinstance(mlp, BloomMLP):
            h1 = K.gelu_tanh(PF.layernorm_linear(x, self.post_attention_layernorm.weight, self.post_attention_layernorm.bias,
                                                 mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias, self.eps, tp))
            return x + F.dropout(PF.linear_residual(h1, mlp.dense_4h_to_h.weight, mlp.dense_4h_to_h.bias, zero, tp), p, True)
        ln = fused_layer_norm(x, self.post_attention_layernorm.weight, self.post_attention_layernorm.bias, self.eps)
        return x + F.dropout(mlp(ln, zero), p, True)

    def forward(self, x: torch.Tensor, batch: int, seq: int, seg_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``x``: ``[tokens_local, hidden]`` (token-sharded when ``self.tp`` is set).  ``seg_start``: int32 ``[batch, seq]``
        document starts of packed rows (``ops.attention``), the same on every tensor-parallel rank; None: one document
        per row."""
        if getattr(self, "fp8", False):
            self._check_fp8()
            return self._forward_fp8(x, batch, seq, seg_start)
        if self.training and (getattr(self, "hidden_dropout", 0.0) > 0.0 or getattr(self, "attention_dropout", 0.0) > 0.0):
            return self._forward_with_dropout(x, batch, seq, seg_start)
        attn = self.self_attention
        tp = self.tp
        n_head_local = attn.query_key_value.weight.shape[0] // (3 * attn.head_dim)
        x = PF.attention_sublayer(x, self.input_layernorm.weight, self.input_layernorm.bias,
                                  attn.query_key_value.weight, attn.query_key_value.bias,
                                  attn.dense.weight, attn.dense.bias, attn.alibi_slopes_local(n_head_local),
                                  self.eps, batch, seq, n_head_local, attn.head_dim, tp, seg_start)
        mlp = self.mlp
        if isinstance(mlp, BloomMLP):
            x = PF.layernorm_mlp(x, self.post_attention_layernorm.weight, self.post_attention_layernorm.bias,
                                 mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias,
                                 mlp.dense_4h_to_h.weight, mlp.dense_4h_to_h.bias, self.eps, tp)
        else:
            # replaced MLP (e.g. ExpertLayer): HF contract mlp(layernorm_output, residual)
            ln = fused_layer_norm(x, self.post_attention_layernorm.weight, self.post_attention_layernorm.bias, self.eps)
            x = mlp(ln, x)
        return x

    def _forward_fp8(self, x: torch.Tensor, batch: int, seq: int, seg_start: Optional[torch.Tensor]) -> torch.Tensor:
        attn, mlp = self.self_attention, self.mlp
        x = PF.attention_sublayer_fp8(x, self.input_layernorm.weight, self.input_layernorm.bias,
                                      attn.query_key_value.weight, attn.query_key_value.bias, attn.dense.weight,
                                      attn.dense.bias, attn.alibi_slopes_local(attn.num_heads), self.eps, batch, seq,
                                      attn.num_heads, attn.head_dim, seg_start)
        return PF.layernorm_mlp_fp8(x, self.post_attention_layernorm.weight, self.post_attention_layernorm.bias,
                                    mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias, mlp.dense_4h_to_h.weight,
                                    mlp.dense_4h_to_h.bias, self.eps)


def _alibi_slopes_local(self: BloomAttention, n_head_local: int) -> torch.Tensor:
    """fp32 slopes of the heads this tensor-parallel rank owns (heads are sharded contiguously);
    kept out of the module's buffers so that ``model.to(bfloat16)`` cannot round them."""
    device = self.query_key_value.weight.device
    key = (n_head_local, str(device))
    slopes = self._slopes_cache.get(key)
    if slopes is None:
        if getattr(self, "use_alibi", True):
            full = K.alibi_slopes(self.num_heads, device=device)
        else:  # no position bias inside attention (learned absolute positions): the flash kernel runs with zero slopes
            full = torch.zeros(self.num_heads, dtype=torch.float32, device=device)
        rank = getattr(self, "tp_rank", 0) if n_head_local != self.num_heads else 0
        slopes = full[rank * n_head_local:(rank + 1) * n_head_local].contiguous()
        self._slopes_cache[key] = slopes
    return slopes


BloomAttention.alibi_slopes_local = _alibi_slopes_local


class _LayerNormFn(torch.autograd.Function):
    """Stand-alone fused LayerNorm (used where the LN is not followed by one of our GEMMs)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        y, mean, rstd = K.layernorm_fwd(x2, gamma, beta, eps)
        ctx.save_for_backward(x2, gamma, beta, mean, rstd)
        ctx.shape = shape
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x2, gamma, beta, mean, rstd = ctx.saved_tensors
        dx, dg, db = PF._ln_bwd(dy.reshape(x2.shape).contiguous(), x2, gamma, beta, mean, rstd)
        return dx.view(ctx.shape), dg, db, None


def fused_layer_norm(x, gamma, beta, eps=1e-5):
    return _LayerNormFn.apply(x, gamma, beta, eps)


def left_align(attention_mask: torch.Tensor):
    """Indices that rotate every row of a ``[batch, seq]`` tensor so that its first real token comes first.

    Returns ``(idx, keep, inverse)``: ``x.gather(1, idx)`` is the left-aligned ``x`` (leading pads wrap around to the
    end), ``keep`` is the rotated mask (``True`` on real tokens) and ``y.gather(1, inverse)`` undoes the rotation.
    Masks with holes (real tokens on both sides of a pad) are refused with a device-side assert — no host sync."""
    m = attention_mask.ne(0)
    S = m.shape[1]
    lead = (m.cumsum(1) == 0).sum(1, keepdim=True)                       # pads in front of the first real token
    pos = torch.arange(S, device=m.device)[None, :]
    idx = (pos + lead) % S
    keep = m.gather(1, idx)
    torch._assert_async((keep[:, :-1] | ~keep[:, 1:]).all(),
                        "pipegoose_b200 models take left- or right-padded batches, not attention masks with holes")
    return idx, keep, (pos - lead) % S


def validate_position_ids(position_ids: torch.Tensor, input_ids: torch.Tensor) -> None:
    """Packed-sequence positions: ``[B, S]`` like ``input_ids``, every row a concatenation of runs ``0, 1, 2, ...``
    (``P[:, 0] == 0``, every step ``+1`` or a reset to 0).  The values are checked with a device-side assert — no host
    sync."""
    if tuple(position_ids.shape) != tuple(input_ids.shape):
        raise ValueError(f"position_ids has shape {tuple(position_ids.shape)}, input_ids {tuple(input_ids.shape)}")
    if position_ids.dtype.is_floating_point or position_ids.dtype == torch.bool:
        raise ValueError(f"position_ids must be an integer tensor, got {position_ids.dtype}")
    P = position_ids
    step = P[:, 1:] - P[:, :-1]
    ok = (P[:, 0] == 0).all() & ((step == 1) | (P[:, 1:] == 0)).all()
    torch._assert_async(ok, "position_ids rows must be runs 0, 1, 2, ... (start at 0; each step +1 or a reset to 0)")


def packed_seg_start(position_ids: torch.Tensor, input_ids: torch.Tensor) -> torch.Tensor:
    """Validated ``position_ids`` -> int32 ``[B, S]`` document starts for the attention kernels."""
    from pipegoose_b200.ops.attention import seg_start_from_position_ids

    validate_position_ids(position_ids, input_ids)
    return seg_start_from_position_ids(position_ids.to(input_ids.device))


def embed_tokens(owner: nn.Module, input_ids: torch.Tensor, config, vocab_start: int, tp,
                 position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Token ids -> ``[tokens_local, hidden]`` input of the first block.  ``owner`` holds ``word_embeddings`` and either
    ``word_embeddings_layernorm`` (Bloom) or ``position_embeddings`` (GPT-2): the model's ``transformer`` or a first
    pipeline stage.  ``position_ids`` (packed rows): the positions learned position embeddings read instead of
    ``arange(S)``; ALiBi models take no positions here."""
    if tp is not None and input_ids.numel() % tp.size != 0:
        raise ValueError(f"the sequence-parallel path shards the {input_ids.numel()} tokens of a batch (batch x seq) over "
                         f"{tp.size} tensor-parallel ranks: pad the batch so that batch x seq is a multiple of {tp.size}")
    if getattr(config, "position_embedding", "alibi") == "learned":
        assert input_ids.shape[-1] <= config.n_positions, "sequence longer than the position table"
        assert not getattr(config, "embedding_layernorm", False)
        return PF.embedding_positions(input_ids, owner.word_embeddings.weight, owner.position_embeddings.weight,
                                      vocab_start, tp, position_ids)
    ln = owner.word_embeddings_layernorm
    return PF.embedding_layernorm(input_ids, owner.word_embeddings.weight, ln.weight, ln.bias,
                                  config.layer_norm_epsilon, vocab_start, tp)


def run_block(block: nn.Module, x: torch.Tensor, batch: int, seq: int, config,
              seg_start: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One transformer block, with activation recomputation when ``config.recompute == "block"`` (training only).
    ``seg_start``: document starts of packed rows (see :meth:`BloomBlock.forward`)."""
    args = (x, batch, seq) if seg_start is None else (x, batch, seq, seg_start)
    if getattr(config, "recompute", "none") == "block" and torch.is_grad_enabled() and x.requires_grad:
        from torch.utils.checkpoint import checkpoint

        return checkpoint(block, *args, use_reentrant=False)
    return block(*args)


class BloomModel(nn.Module):
    def __init__(self, config: BloomConfig):
        super().__init__()
        h = config.hidden_size
        self.config = config
        self.word_embeddings = nn.Embedding(config.vocab_size, h)
        if config.embedding_layernorm:
            self.word_embeddings_layernorm = nn.LayerNorm(h, eps=config.layer_norm_epsilon)
        if config.position_embedding == "learned":
            assert config.n_positions > 0, "learned position embeddings need n_positions"
            self.position_embeddings = nn.Embedding(config.n_positions, h)
        self.h = nn.ModuleList([BloomBlock(config) for _ in range(config.n_layer)])
        self.ln_f = nn.LayerNorm(h, eps=config.layer_norm_epsilon)


def filter_logits(logits: torch.Tensor, temperature: float, top_k: int, top_p: float) -> torch.Tensor:
    """The sampling distribution's logits: ``logits [B, V]`` scaled by ``1 / temperature``, then everything outside the
    top ``top_k`` and outside the nucleus of mass ``top_p`` set to ``-inf``.  Its softmax is what sampling draws from."""
    if temperature != 1.0:
        logits = logits / max(float(temperature), 1e-6)
    if top_k and top_k > 0:
        kth = logits.topk(min(int(top_k), logits.shape[-1]), dim=-1).values[:, -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if top_p < 1.0:
        sorted_logits, order = logits.sort(dim=-1, descending=True)
        probs = sorted_logits.softmax(-1)
        # drop a token when the mass BEFORE it already reaches top_p (the most likely token always stays)
        drop = (probs.cumsum(-1) - probs) >= top_p
        sorted_logits = sorted_logits.masked_fill(drop, float("-inf"))
        logits = torch.full_like(logits, float("-inf")).scatter(-1, order, sorted_logits)
    return logits


class BloomForCausalLM(nn.Module):
    base_model_prefix = "transformer"

    def __init__(self, config: BloomConfig):
        super().__init__()
        assert not config.apply_residual_connection_post_layernorm
        self.config = config
        self.transformer = BloomModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.lm_head.weight = self.transformer.word_embeddings.weight  # tied
        # the tied table receives two gradient contributions per backward (lm_head wgrad + embedding
        # scatter): the gradient reducer must wait for both before reducing its bucket
        self.lm_head.weight._pg_grad_contribs = 2
        self.tp = None
        self.vocab_start = 0
        self.apply(self._init_weights)

    def _init_weights(self, module):
        std = self.config.initializer_range
        if isinstance(module, nn.Linear):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.Embedding):
            module.weight.data.normal_(mean=0.0, std=std)
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    # ------------------------------------------------------------------ helpers
    def get_input_embeddings(self):
        return self.transformer.word_embeddings

    def get_output_embeddings(self):
        return self.lm_head

    def num_parameters(self) -> int:
        seen, n = set(), 0
        for p in self.parameters():
            if id(p) not in seen:
                seen.add(id(p))
                n += p.numel()
        return n

    def flops_per_token(self, seq_len: int) -> float:
        """Model FLOPs per token for fwd+bwd (6*N_matmul + causal attention)."""
        c = self.config
        h, L, V = c.hidden_size, c.n_layer, c.vocab_size
        per_layer = 12 * h * h
        attn = 2 * seq_len * h  # QK^T + PV, causal half of 4*S*h
        return 3 * 2 * (L * (per_layer + attn) + V * h)

    # ------------------------------------------------------------------ forward
    def hidden_states(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor] = None,
                      seg_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``position_ids``: packed rows (see :meth:`forward`); ``seg_start``: their document starts when the caller
        already derived them (:func:`packed_seg_start`)."""
        t = self.transformer
        B, S = input_ids.shape
        if position_ids is not None and seg_start is None:
            seg_start = packed_seg_start(position_ids, input_ids)
        x = embed_tokens(t, input_ids, self.config, self.vocab_start, self.tp, position_ids)
        for block in t.h:
            x = run_block(block, x, B, S, self.config, seg_start)
        return x

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                labels: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                **_unused) -> CausalLMOutput:
        """``position_ids`` (``[B, S]``, packed sequences, as 🤗's ``DataCollatorWithFlattening`` emits them): every row
        is a concatenation of documents, each numbered ``0, 1, 2, ...``.  Tokens attend only within their document,
        learned position embeddings read these positions, and a document's last token has no target (the next
        document's first token is not predicted).  The result equals running every document as its own sequence, with
        the loss averaged over all documents' target tokens.  Not combined with an ``attention_mask`` that has zeros:
        pad the tail of a packed row as one more document with ``-100`` labels instead."""
        t = self.transformer
        B, S = input_ids.shape
        unroll = None
        seg_start = None
        if position_ids is not None:
            if attention_mask is not None and bool((attention_mask == 0).any()):
                raise ValueError("position_ids (packed sequences) cannot be combined with an attention_mask that has "
                                 "zeros: pad the tail of a packed row as one more document with -100 labels instead")
            attention_mask = None
            position_ids = position_ids.to(input_ids.device)
            seg_start = packed_seg_start(position_ids, input_ids)
        if attention_mask is not None:
            # The fused attention is purely causal.  RIGHT padding is harmless under a causal mask (real tokens never
            # attend to later pads).  LEFT padding (what 🤗's Bloom tokenizer produces) is turned into right padding by
            # rotating every row until its first real token sits at position 0: ALiBi only sees distances between real
            # tokens, so their hidden states are what 🤗 computes with the mask.  Pads never count in the loss.
            idx, keep, unroll = left_align(attention_mask)
            input_ids = input_ids.gather(1, idx)
            if labels is not None:
                labels = labels.gather(1, idx).masked_fill(~keep, -100)
        x = self.hidden_states(input_ids, position_ids, seg_start)
        eps = self.config.layer_norm_epsilon
        if labels is not None:
            # HF semantics: position s predicts token s+1; the last position has no target
            shifted = torch.full_like(labels, -100)
            shifted[:, :-1] = labels[:, 1:]
            if position_ids is not None:   # nor does the last token of a packed document
                shifted[:, :-1].masked_fill_(position_ids[:, 1:] == 0, -100)
            loss = PF.lm_head_cross_entropy(x, t.ln_f.weight, t.ln_f.bias, self.lm_head.weight, shifted, eps,
                                            self.vocab_start, -100, self.tp, vocab_size=self.config.vocab_size)
            return CausalLMOutput(loss=loss, logits=None)
        ln = fused_layer_norm(x, t.ln_f.weight, t.ln_f.bias, eps)
        if self.tp is not None:
            ln = self.tp.gather_rows(ln)
        logits = PF.linear(ln, self.lm_head.weight)
        if self.tp is not None:
            logits = self.tp.gather_cols(logits)[:, : self.config.vocab_size]
        logits = logits.view(B, S, -1)
        if unroll is not None:   # back to the caller's layout (pad positions hold the logits of the rotated pads)
            logits = logits.gather(1, unroll[:, :, None].expand(-1, -1, logits.shape[-1]))
        return CausalLMOutput(loss=None, logits=logits)

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, max_new_tokens: int = 1, use_cache: bool = True,
                 attention_mask: Optional[torch.Tensor] = None, do_sample: bool = False, temperature: float = 1.0,
                 top_k: int = 0, top_p: float = 1.0, eos_token_id: Optional[int] = None,
                 pad_token_id: Optional[int] = None, generator: Optional[torch.Generator] = None, **_unused) -> torch.Tensor:
        """Decoding with 🤗 ``generate``'s vocabulary for the common cases: greedy by default, ``do_sample`` with
        ``temperature`` / ``top_k`` / ``top_p``; rows stop at ``eos_token_id`` (later positions hold ``pad_token_id``,
        default: the eos id) and the loop ends when every row has stopped; returns ``input_ids`` followed by the new
        tokens.  Under tensor parallelism every rank returns the same tokens (sampled on the group's first rank).

        ``use_cache``: keys and values of every layer are kept — under tensor parallelism each rank caches the heads it
        owns — the prompt is processed once and each new token costs one position.  Mixture-of-experts blocks
        (``ExpertLayer``) decode incrementally too: the router sees the new positions only (an expert-capacity limit
        then counts the tokens of one decoding step, not of the whole sequence — with a limit that binds, cached and
        uncached decoding may drop different tokens).  🤗's left-padded prompts of unequal length (``attention_mask`` with
        leading zeros) are cached too: pad keys are masked per row, ALiBi only sees distances between real tokens.
        Masks that are not left-padded are refused (the new tokens go behind the last column).  On CUDA bf16 models whose
        head size is 64, 80 or 128 the cache is preallocated for ``prompt + max_new_tokens`` positions, the prompt runs
        through the flash kernel and every new token through the split-KV decode kernel.  Recomputed through the
        training forward for every token instead: models with a fused NVLink MoE layer (kernels built around
        token-sharded full sequences), ``use_cache=False``, and pipelined models (``PipelineParallel``: one forward-only
        schedule per token, the last stage picks the token and broadcasts it to the other stages)."""
        B, prompt_len = input_ids.shape
        ragged = attention_mask is not None and bool((attention_mask == 0).any())
        dense = all(isinstance(b.mlp, BloomMLP) or _decodes_incrementally(b.mlp) for b in self.transformer.h)
        group = self.tp.size if self.tp is not None else 1
        mask = attention_mask.to(input_ids.device).long() if ragged else None
        lead = None
        if ragged:
            # pads in front of each row; the KV-cache path takes LEFT-padded prompts (every row: zeros, then ones)
            lead = (mask.cumsum(1) == 0).sum(1)
            if not bool((mask.sum(1) + lead == prompt_len).all()):
                raise ValueError("generate() takes LEFT-padded prompts (attention_mask rows: zeros, then ones): new tokens "
                                 "are appended behind the last column, which must be every row's last real token")
        # a pipelined model (PipelineParallel): every new token is one forward-only schedule through the stages — keys and
        # values are not cached across stages — and the last stage, which holds the logits, tells the others the token
        engine = getattr(self, "_pg_pipeline_engine", None)
        cached = use_cache and dense and engine is None
        out = input_ids
        finished = torch.zeros(B, dtype=torch.bool, device=input_ids.device)
        fill = pad_token_id if pad_token_id is not None else (eos_token_id if eos_token_id is not None else 0)
        cache = [None] * len(self.transformer.h)
        for step in range(max_new_tokens):
            if cached:
                last = self._incremental_logits(out if step == 0 else out[:, -1:], cache,
                                                0 if step == 0 else out.shape[1] - 1, lead,
                                                capacity=prompt_len + max_new_tokens)[:, -1, :]
            else:
                S = out.shape[1]
                pad = 0
                # token-sharded activations need a multiple of the group size (per micro-batch under a pipeline engine:
                # whole rows, so the row length itself is padded)
                while ((S + pad) if engine is not None else (B * (S + pad))) % group:
                    pad += 1
                if ragged:   # pads go in FRONT (mask 0): the batch stays left-padded, the last column the newest token
                    ids = out if pad == 0 else torch.cat([out.new_zeros(B, pad), out], dim=1)
                    m = mask if pad == 0 else torch.cat([mask.new_zeros(B, pad), mask], dim=1)
                    pos = -1
                else:        # right padding is harmless under a causal mask
                    ids = out if pad == 0 else torch.cat([out, out.new_zeros(B, pad)], dim=1)
                    m, pos = None, S - 1
                if engine is None:
                    last = (self(ids, attention_mask=m) if m is not None else self(ids)).logits[:, pos, :]
            if engine is not None:
                nxt = self._pipelined_next_token(engine, ids, m, pos, lambda logits: self._select_token(
                    logits, do_sample, temperature, top_k, top_p, generator))
            else:
                nxt = self._select_token(last.float(), do_sample, temperature, top_k, top_p, generator)
            if eos_token_id is not None:
                nxt = torch.where(finished, torch.full_like(nxt, fill), nxt)
                finished = finished | (nxt == eos_token_id)
            out = torch.cat([out, nxt[:, None]], dim=1)
            if ragged:
                mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
            if eos_token_id is not None and bool(finished.all()):
                break
        return out

    def _pipelined_next_token(self, engine, ids: torch.Tensor, mask: Optional[torch.Tensor], pos: int, select) -> torch.Tensor:
        """One decoding step of a pipelined model: a forward-only schedule (micro-batched like training), the token chosen
        on the last stage from the logits at ``pos`` and broadcast over the PIPELINE group."""
        import torch.distributed as dist

        from pipegoose_b200.distributed.parallel_mode import ParallelMode

        outs = self(ids, attention_mask=mask) if mask is not None else self(ids)
        if not all(isinstance(b.mlp, BloomMLP) for b in self.transformer.h):
            # mixture-of-experts stages push their router losses on every forward: nothing consumes them while decoding
            from pipegoose_b200.nn.expert_parallel.expert_context import ExpertContext

            store = ExpertContext.get_instance()
            store.pop_all_aux_loss(), store.pop_all_z_loss()
        ctx = engine.parallel_context
        if engine.is_last:
            logits = torch.cat([o.logits if hasattr(o, "logits") else o for o in outs], dim=0)
            nxt = select(logits[:, pos, :].float())
        else:
            nxt = torch.empty(ids.shape[0], dtype=torch.long, device=ids.device)
        dist.broadcast(nxt, src=ctx.get_ranks_in_group(ParallelMode.PIPELINE)[-1], group=ctx.get_group(ParallelMode.PIPELINE))
        return nxt

    def _select_token(self, logits: torch.Tensor, do_sample: bool, temperature: float, top_k: int, top_p: float,
                      generator: Optional[torch.Generator]) -> torch.Tensor:
        """Next token of every row from its fp32 logits ``[B, V]``: arg-max, or a sample from the (temperature-scaled,
        top-k / nucleus-filtered) distribution.  Sampled tokens are made identical on every tensor-parallel rank."""
        if not do_sample:
            return logits.argmax(-1)
        nxt = torch.multinomial(filter_logits(logits, temperature, top_k, top_p).softmax(-1), 1,
                                generator=generator).squeeze(-1)
        if self.tp is not None and self.tp.size > 1:
            import torch.distributed as dist

            dist.broadcast(nxt, src=dist.get_global_rank(self.tp.group, 0), group=self.tp.group)
        return nxt

    def _incremental_logits(self, ids: torch.Tensor, cache: list, past: int,
                            lead: Optional[torch.Tensor] = None, capacity: Optional[int] = None) -> torch.Tensor:
        """Inference-only forward of ``ids`` (positions ``past .. past+T-1``) against the cached keys / values; plain
        tensor ops on the module's weights (the fused training kernels are built around full sequences).  ``lead[b]``:
        number of pad positions in front of row ``b`` (left-padded batch; None: no pads) — pad keys are masked with a
        large finite negative (a pad QUERY then attends uniformly instead of producing NaNs that ``0 * NaN`` would
        carry into real rows), learned absolute positions count from the first real token.  ALiBi needs no shift:
        ``slope * key_position`` differs from 🤗's mask-derived bias by a per-row constant, which softmax ignores.

        CUDA bf16 models whose head size has a decode kernel run attention natively instead (:func:`_cached_attention`):
        the keys / values live in buffers of ``capacity`` positions (default: the prompt length) allocated at the
        prompt, which goes through the flash kernel; every later call appends one position."""
        t, cfg = self.transformer, self.config
        B, T = ids.shape
        h, n_head = cfg.hidden_size, cfg.n_head
        D = h // n_head
        tp = self.tp
        if tp is not None:
            return self._incremental_logits_tp(ids, cache, past, lead, capacity)
        native = _native_decode(t.h[0].self_attention.query_key_value.weight, D)
        if native and lead is not None:
            lead = lead.to(torch.int32)          # the kernels' type, converted once for every layer
        positions = _learned_positions(t.position_embeddings.weight, past, T, lead) if _learned(cfg) else None

        def attend(li, attn, qkv):
            if native:
                return _cached_attention(qkv, attn.alibi_slopes_local(n_head), cache, li, past, lead, capacity, n_head, D)
            qkv = qkv.view(B, T, n_head, 3, D)
            q, k, v = (qkv[:, :, :, i].transpose(1, 2) for i in range(3))               # [B, H, T, D]
            if cache[li] is not None:
                k, v = torch.cat([cache[li][0], k], dim=2), torch.cat([cache[li][1], v], dim=2)
            cache[li] = (k, v)
            S = k.shape[2]
            scores = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(D)   # [B, H, T, S]
            key_pos = torch.arange(S, device=ids.device, dtype=torch.float32)
            if attn.use_alibi:
                scores = scores + K.alibi_slopes(n_head, device=ids.device).view(1, n_head, 1, 1) * key_pos
            query_pos = torch.arange(past, past + T, device=ids.device).view(T, 1)
            scores = scores.masked_fill(key_pos.view(1, S) > query_pos, float("-inf"))
            scores = _mask_leading_pads(scores, key_pos, lead)
            return torch.matmul(scores.softmax(-1).to(v.dtype), v).transpose(1, 2).reshape(B, T, h)

        x = self._inference_layers(self._inference_embed(ids, positions), attend)
        return self._inference_head(x[:, -1:])

    def _inference_embed(self, ids: torch.Tensor, positions: Optional[torch.Tensor]) -> torch.Tensor:
        """Token embeddings of the inference-only forwards: plus ``positions`` (rows of the learned position table) on
        GPT-2-style models, the embedding LayerNorm on Bloom."""
        import torch.nn.functional as F

        t, cfg = self.transformer, self.config
        x = F.embedding(ids, t.word_embeddings.weight)
        if _learned(cfg):
            return x + positions
        return F.layer_norm(x, (cfg.hidden_size,), t.word_embeddings_layernorm.weight, t.word_embeddings_layernorm.bias,
                            cfg.layer_norm_epsilon)

    def _inference_layers(self, x: torch.Tensor, attend) -> torch.Tensor:
        """Every block of an inference-only forward on ``x [B, T, h]``: plain tensor ops on the module's weights (the
        fused training kernels are built around full sequences).  ``attend(li, attn, qkv)`` is the attention of layer
        ``li`` (``attn``: its ``BloomAttention``), from ``qkv [B, T, n_head*3*D]`` to ``[B, T, n_head*D]``; it is the only
        step the KV-cached and the paged forwards do differently."""
        import torch.nn.functional as F

        h = self.config.hidden_size
        for li, block in enumerate(self.transformer.h):
            attn = block.self_attention
            ln = F.layer_norm(x, (h,), block.input_layernorm.weight, block.input_layernorm.bias, block.eps)
            qkv = F.linear(ln, attn.query_key_value.weight, attn.query_key_value.bias)
            x = x + F.linear(attend(li, attn, qkv), attn.dense.weight, attn.dense.bias)
            ln = F.layer_norm(x, (h,), block.post_attention_layernorm.weight, block.post_attention_layernorm.bias, block.eps)
            mlp = block.mlp
            if not isinstance(mlp, BloomMLP):
                x = _moe_on_replicated_tokens(mlp, ln, x)
                continue
            x = x + F.linear(K.gelu_tanh(F.linear(ln, mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias)),
                             mlp.dense_4h_to_h.weight, mlp.dense_4h_to_h.bias)
        return x

    def _inference_head(self, x: torch.Tensor) -> torch.Tensor:
        """Final LayerNorm and lm_head of the inference-only forwards."""
        import torch.nn.functional as F

        t, cfg = self.transformer, self.config
        x = F.layer_norm(x, (cfg.hidden_size,), t.ln_f.weight, t.ln_f.bias, cfg.layer_norm_epsilon)
        return F.linear(x, self.lm_head.weight)

    @torch.no_grad()
    def _paged_logits(self, ids: torch.Tensor, positions: torch.Tensor, k_pools: torch.Tensor, v_pools: torch.Tensor,
                      seg_start: Optional[torch.Tensor] = None, slot: Optional[torch.Tensor] = None,
                      last: Optional[torch.Tensor] = None, table: Optional[torch.Tensor] = None,
                      max_pos: int = 0, cu_seqlens: Optional[torch.Tensor] = None,
                      start: Optional[torch.Tensor] = None, max_len: int = 0,
                      k_scales: Optional[torch.Tensor] = None, v_scales: Optional[torch.Tensor] = None,
                      stage: Optional[tuple] = None, n_dec: Optional[int] = None) -> torch.Tensor:
        """Inference-only forward of a set of sequences over paged KV pools (``pipegoose_b200.serving``); ``ids`` and
        ``positions`` (each token's position in its own sequence) are ``[N]``, ``k_pools`` / ``v_pools`` are
        ``[n_layer, num_pages, n_head, 64, D]``.  Three modes:

        - prefill (``seg_start`` given): the prompts packed into one row, each a document of the flash kernel's
          ``seg_start`` (int32 ``[N]``); ``slot`` (int32 ``[N]``) is each token's pool slot (``page * 64 + offset``).
          Returns the logits at the tokens ``last`` (``[n]``, each prompt's last token): ``[n, V]``.
        - decode: one new token per sequence; ``table`` (int32 ``[N, max_pages]``) holds each sequence's pages,
          ``positions`` (int32) its new token's position, ``max_pos >= max(positions)``.  Returns ``[N, V]``.
        - prefill with cached prefixes (``start`` given): the suffixes of R prompts whose first ``start[r]`` positions
          are already in the pools, packed back to back (sequence r: tokens ``cu_seqlens[r] .. cu_seqlens[r+1]-1``);
          ``positions`` are absolute, ``slot`` is each token's pool slot, ``table`` (int32 ``[R, max_pages]``) each
          sequence's pages and ``max_len >=`` its suffix length.  Every layer stores the new keys and values, then the
          suffix attends to the whole sequence through the pools.  Returns the logits at ``last``: ``[R, V]``.
        - append (``cu_seqlens`` given without ``start``): R sequences append 1 .. ``APPEND_MAX_TOKENS`` tokens each,
          packed back to back as above; ``positions`` are absolute, ``table`` (int32 ``[R, max_pages]``) holds each
          sequence's pages, ``max_pos >=`` every appended position and ``max_len >=`` every sequence's appended
          tokens (0: derived, see ``alibi_paged_append_attention``).  Every layer writes the new keys and values and
          attends through the paged append-attention op.  Returns the logits of every token: ``[N, V]``.
        - mixed (``n_dec`` given, chunked prefill): ``n_dec`` decode tokens (one per sequence, as in decode mode)
          followed by prompt chunks of R sequences (as in the prefill with cached prefixes: ``cu_seqlens`` counts the
          chunk rows from 0, ``start[r]`` is chunk r's first position, ``slot`` holds the chunk tokens' pool slots).
          ``table`` (int32 ``[n_dec + R, max_pages]``) holds the decode rows' pages, then the chunks'; ``max_pos`` bounds
          the decode positions and ``max_len`` the chunk lengths.  Every layer runs the decode rows through the paged
          decode op (which writes their keys and values), writes the chunks' keys and values and runs the chunks
          through the paged prefill op; the two touch disjoint pages.  Returns the logits at the rows ``last`` (indices
          into all N rows): ``[len(last), V]``.

        FP8 pools (``float8_e4m3fn``) come with fp32 ``k_scales`` / ``v_scales`` ``[n_layer, num_pages, n_head, 64]``;
        a prefill with cached prefixes then also takes ``stage = (num_pages, src, dst, slot, table)``, the device form of
        :func:`~pipegoose_b200.ops.attention.fp8_prefill_staging` (``table`` as ``[R, width]``), which the kernel path
        reads through one bf16 staging pool shared by all layers (the paged prefill op refuses FP8 pools without it);
        so does the mixed mode, for its chunks.

        CUDA bf16 models with head size 64, 80 or 128 run the flash / paged decode / paged prefill / append kernels;
        otherwise (CPU, fp32, other head sizes) their PyTorch references run, over FP8 pools too (append: not over FP8
        pools)."""
        from pipegoose_b200.ops import attention as A

        cfg = self.config
        n_head = cfg.n_head
        D = cfg.hidden_size // n_head
        N = ids.shape[0]
        native = _native_decode(self.transformer.h[0].self_attention.query_key_value.weight, D)
        write = A.paged_kv_write if native else A.paged_kv_write_reference
        decode = A.alibi_paged_decode_attention if native else A.alibi_paged_decode_attention_reference
        prefill = A.alibi_paged_prefill_attention if native else A.paged_prefill_attention_fp32
        append = A.alibi_paged_append_attention if native else A.alibi_paged_append_attention_reference
        pos_emb = self.transformer.position_embeddings.weight[positions.long()] if _learned(cfg) else None
        # append: each sequence's first new position
        first = positions[cu_seqlens[:-1].long()] if cu_seqlens is not None and start is None else None
        staging = None
        if native and k_scales is not None and stage is not None:
            shape = (stage[0], n_head, A.PAGE_SIZE, D)
            w = self.transformer.h[0].self_attention.query_key_value.weight
            staging = (w.new_empty(shape), w.new_empty(shape)) + tuple(stage[1:])

        def attend(li, attn, qkv):
            qkv = qkv.view(N, n_head * 3 * D)
            slopes = attn.alibi_slopes_local(n_head)
            scales = {} if k_scales is None else {"k_scales": k_scales[li], "v_scales": v_scales[li]}
            if seg_start is not None:
                write(qkv, slot, k_pools[li], v_pools[li], D, **scales)
                return A.alibi_attention(qkv, slopes, 1, N, n_head, D, seg_start=seg_start.view(1, N)).view(1, N, -1)
            if n_dec is not None:
                dec, new = qkv[:n_dec], qkv[n_dec:]
                write(new, slot, k_pools[li], v_pools[li], D, **scales)
                chunk = dict(scales, stage=staging) if staging is not None else scales
                args = (new, k_pools[li], v_pools[li], table[n_dec:], cu_seqlens, start, max_len, slopes, D)
                dec_args = (dec, k_pools[li], v_pools[li], table[:n_dec], positions[:n_dec], max_pos, slopes, D)
                if not native:                                   # the references
                    out = prefill(*args, **chunk)
                    return (torch.cat([decode(*dec_args, **scales), out]) if n_dec else out).view(1, N, -1)
                out = qkv.new_empty(N, n_head * D)               # both kernels write their rows of one buffer
                prefill(*args, out=out[n_dec:], **chunk)
                if n_dec:
                    decode(*dec_args, out=out[:n_dec], **scales)
                return out.view(1, N, -1)
            if start is not None:
                write(qkv, slot, k_pools[li], v_pools[li], D, **scales)
                if staging is not None:
                    scales["stage"] = staging
                return prefill(qkv, k_pools[li], v_pools[li], table, cu_seqlens, start, max_len, slopes, D,
                               **scales).view(1, N, -1)
            if cu_seqlens is not None:
                return append(qkv, k_pools[li], v_pools[li], table, cu_seqlens, first, max_pos, slopes, D,
                              max_tokens=max_len).view(1, N, -1)
            return decode(qkv, k_pools[li], v_pools[li], table, positions, max_pos, slopes, D, **scales).view(1, N, -1)

        x = self._inference_layers(self._inference_embed(ids.view(1, N), pos_emb), attend)[0]
        return self._inference_head(x if last is None else x[last.long()])

    def _incremental_logits_tp(self, ids: torch.Tensor, cache: list, past: int,
                               lead: Optional[torch.Tensor] = None, capacity: Optional[int] = None) -> torch.Tensor:
        """:meth:`_incremental_logits` on a tensor-parallel model: activations are replicated ``[B, T, h]`` (decoding is
        latency-bound: no sequence sharding), every rank runs the attention heads / MLP columns / vocabulary rows it owns
        and caches ITS heads' keys and values; row-parallel products and the embedding are summed over the group, the
        last position's logits are gathered along the vocabulary."""
        import torch.distributed as dist
        import torch.nn.functional as F

        t, cfg, tp = self.transformer, self.config, self.tp
        group, rank, world = tp.group, tp.rank, tp.size
        B, T = ids.shape
        h = cfg.hidden_size
        D = h // cfg.n_head
        native = _native_decode(t.h[0].self_attention.query_key_value.weight, D)
        if native and lead is not None:
            lead = lead.to(torch.int32)

        def all_reduce(x):
            dist.all_reduce(x, group=group)
            return x

        table = t.word_embeddings.weight                      # [V_padded / world, h]
        local = ids - self.vocab_start
        mine = (local >= 0) & (local < table.shape[0])
        x = F.embedding(local.clamp(0, table.shape[0] - 1), table) * mine.unsqueeze(-1).to(table.dtype)
        x = all_reduce(x)
        if getattr(cfg, "position_embedding", "alibi") == "learned":
            x = x + _learned_positions(t.position_embeddings.weight, past, T, lead)
        else:
            x = F.layer_norm(x, (h,), t.word_embeddings_layernorm.weight, t.word_embeddings_layernorm.bias, cfg.layer_norm_epsilon)
        for li, block in enumerate(t.h):
            attn, mlp = block.self_attention, block.mlp
            n_local = attn.query_key_value.weight.shape[0] // (3 * D)
            ln = F.layer_norm(x, (h,), block.input_layernorm.weight, block.input_layernorm.bias, block.eps)
            qkv = F.linear(ln, attn.query_key_value.weight, attn.query_key_value.bias)
            if native:
                ctx = _cached_attention(qkv, attn.alibi_slopes_local(n_local), cache, li, past, lead, capacity, n_local, D)
            else:
                qkv = qkv.view(B, T, n_local, 3, D)
                q, k, v = (qkv[:, :, :, i].transpose(1, 2) for i in range(3))               # [B, H/world, T, D]
                if cache[li] is not None:
                    k, v = torch.cat([cache[li][0], k], dim=2), torch.cat([cache[li][1], v], dim=2)
                cache[li] = (k, v)
                S = k.shape[2]
                scores = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(D)
                key_pos = torch.arange(S, device=ids.device, dtype=torch.float32)
                scores = scores + attn.alibi_slopes_local(n_local).view(1, n_local, 1, 1) * key_pos
                query_pos = torch.arange(past, past + T, device=ids.device).view(T, 1)
                scores = scores.masked_fill(key_pos.view(1, S) > query_pos, float("-inf"))
                scores = _mask_leading_pads(scores, key_pos, lead)
                ctx = torch.matmul(scores.softmax(-1).to(v.dtype), v).transpose(1, 2).reshape(B, T, n_local * D)
            x = x + all_reduce(F.linear(ctx, attn.dense.weight)) + attn.dense.bias      # row-parallel: bias once
            ln = F.layer_norm(x, (h,), block.post_attention_layernorm.weight, block.post_attention_layernorm.bias, block.eps)
            if not isinstance(mlp, BloomMLP):
                x = _moe_on_replicated_tokens(mlp, ln, x)    # experts sharded over the group: the layer all-reduces
                continue
            h1 = K.gelu_tanh(F.linear(ln, mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias))
            x = x + all_reduce(F.linear(h1, mlp.dense_4h_to_h.weight)) + mlp.dense_4h_to_h.bias
        x = F.layer_norm(x[:, -1:], (h,), t.ln_f.weight, t.ln_f.bias, cfg.layer_norm_epsilon)
        part = F.linear(x, self.lm_head.weight).contiguous()                            # [B, 1, V_padded / world]
        parts = [torch.empty_like(part) for _ in range(world)]
        dist.all_gather(parts, part, group=group)
        return torch.cat(parts, dim=-1)[..., : cfg.vocab_size]

    # ------------------------------------------------------------------ HF interop
    @classmethod
    def from_hf(cls, hf_model) -> "BloomForCausalLM":
        model = cls(BloomConfig.from_hf(hf_model.config))
        model.load_state_dict(hf_model.state_dict(), strict=False)
        return model

    def to_hf(self):
        """A 🤗 ``transformers.BloomForCausalLM`` with this model's weights (the way back from :meth:`from_hf` / the
        in-place conversion of ``TensorParallel``): parameter names are the same, so this is a config translation and a
        ``load_state_dict``.  The model must be whole — ``deparallelize()`` a live tensor- / pipeline-parallel model
        first, or merge its checkpoint with ``nn.checkpoint_convert`` and load that."""
        from transformers import BloomForCausalLM as HFBloom

        if self.tp is not None or getattr(self, "_pg_pipeline_engine", None) is not None:
            raise ValueError("to_hf() needs the unsharded model: deparallelize() first (or consolidate the checkpoint)")
        if getattr(self.config, "position_embedding", "alibi") != "alibi":
            raise ValueError("to_hf() exports Bloom-architecture models (GPT-2 family: GPT2LMHeadModel.to_hf_state_dict)")
        hf = HFBloom(getattr(self, "hf_config", None) or self.config.to_hf())
        hf = hf.to(next(self.parameters()).dtype)
        missing, unexpected = hf.load_state_dict(self.state_dict(), strict=False)
        assert not unexpected and all("lm_head" in k for k in missing), (missing, unexpected)      # (tied head)
        hf.tie_weights()
        return hf

    def save_hf_pretrained(self, path: str, **kwargs) -> None:
        """``to_hf().save_pretrained(path)``: a directory 🤗 ``from_pretrained`` reads (config.json + weights)."""
        self.to_hf().save_pretrained(path, **kwargs)


def _learned(cfg) -> bool:
    """Learned absolute position embeddings (GPT-2) rather than ALiBi?"""
    return getattr(cfg, "position_embedding", "alibi") == "learned"


def _native_decode(qkv_weight: torch.Tensor, D: int) -> bool:
    """Does KV-cached decoding run attention on the sm_90a kernels (CUDA bf16 weights, a head size the decode kernel
    has)?  Otherwise the eager attention of ``_incremental_logits`` runs."""
    from pipegoose_b200.ops import use_native
    from pipegoose_b200.ops.attention import DECODE_HEAD_DIMS

    return use_native(qkv_weight) and D in DECODE_HEAD_DIMS


def _cached_attention(qkv: torch.Tensor, slopes: torch.Tensor, cache: list, li: int, past: int,
                      lead: Optional[torch.Tensor], capacity: Optional[int], n_head: int, D: int) -> torch.Tensor:
    """Native attention of layer ``li`` for ``qkv [B, T, n_head*3*D]`` at positions ``past .. past+T-1``: the prompt
    (``past == 0``) through the flash kernel, whose document starts express the left pads (a real token of row b sees
    keys from ``lead[b]`` on, a pad sees the pads in front of it), then copied once into fresh ``[B, n_head, capacity,
    D]`` buffers; one new position (``T == 1``) through the split-KV decode kernel, which appends to them.
    ``cache[li]`` is ``(k[:, :, :filled], v[:, :, :filled], k_buffer, v_buffer)``.  Returns ``[B, T, n_head*D]``."""
    from pipegoose_b200.ops.attention import alibi_attention, alibi_decode_attention

    B, T = qkv.shape[:2]
    if past == 0 and cache[li] is None:
        capacity = T if capacity is None else capacity
        if capacity < T:
            raise ValueError(f"KV cache capacity {capacity} is smaller than the prompt ({T} positions)")
        seg = None
        if lead is not None:
            s = torch.arange(T, device=qkv.device).view(1, T)
            first = lead.view(B, 1).to(s.dtype)
            seg = torch.where(s >= first, first, torch.zeros_like(first)).to(torch.int32)
        ctx = alibi_attention(qkv.reshape(B * T, -1), slopes, B, T, n_head, D, seg_start=seg)
        kv = qkv.view(B, T, n_head, 3, D)
        k_buf = qkv.new_empty(B, n_head, capacity, D)
        v_buf = qkv.new_empty(B, n_head, capacity, D)
        k_buf[:, :, :T].copy_(kv[:, :, :, 1].transpose(1, 2))
        v_buf[:, :, :T].copy_(kv[:, :, :, 2].transpose(1, 2))
        cache[li] = (k_buf[:, :, :T], v_buf[:, :, :T], k_buf, v_buf)
        return ctx.view(B, T, n_head * D)
    if T != 1 or cache[li] is None or cache[li][0].shape[2] != past:
        raise ValueError(f"the native KV cache takes a prompt at position 0 and then one token per call "
                         f"(got {T} positions at {past})")
    k_buf, v_buf = cache[li][2], cache[li][3]
    if past >= k_buf.shape[2]:
        raise ValueError(f"KV cache full: position {past} is past its capacity of {k_buf.shape[2]}")
    ctx = alibi_decode_attention(qkv.view(B, -1), k_buf, v_buf, slopes, past, lead, D)
    cache[li] = (k_buf[:, :, :past + 1], v_buf[:, :, :past + 1], k_buf, v_buf)
    return ctx.view(B, 1, n_head * D)


def _mask_leading_pads(scores: torch.Tensor, key_pos: torch.Tensor, lead: Optional[torch.Tensor]) -> torch.Tensor:
    """``scores [B, H, T, S]``: keys in front of row ``b``'s first real token (``key_pos < lead[b]``) get the most
    negative finite value."""
    if lead is None:
        return scores
    pad = key_pos.view(1, 1, 1, -1) < lead.view(-1, 1, 1, 1).to(key_pos.dtype)
    return scores.masked_fill(pad, torch.finfo(scores.dtype).min)


def _learned_positions(table: torch.Tensor, past: int, T: int, lead: Optional[torch.Tensor]) -> torch.Tensor:
    """Rows of a learned absolute position table for raw positions ``past .. past+T-1``; with left padding a row's
    positions count from its first real token (pads read position 0)."""
    if lead is None:
        return table[past:past + T]
    pos = (torch.arange(past, past + T, device=table.device).view(1, T) - lead.view(-1, 1)).clamp(min=0)
    return table[pos]


def _decodes_incrementally(mlp: nn.Module) -> bool:
    """Can this replaced MLP run on a few replicated positions (``mlp(layernorm_output, residual)``)?  ``ExpertLayer``
    can (router + experts on whatever tokens it is given); the fused NVLink MoE layer cannot."""
    from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer

    return type(mlp) is ExpertLayer


def _moe_on_replicated_tokens(mlp: nn.Module, ln: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
    """One decoding step through an ``ExpertLayer``: activations are replicated over the tensor group while decoding, so
    the layer runs in its replicated-token layout (every rank routes all positions, applies the experts it owns, the
    partial outputs are all-reduced) whatever layout training uses; the router's auxiliary terms are discarded."""
    from pipegoose_b200.nn.expert_parallel.expert_context import ExpertContext

    store = ExpertContext.get_instance()
    kept_aux, kept_z = store.pop_all_aux_loss(), store.pop_all_z_loss()
    comm = getattr(mlp, "token_comm", None)
    mlp.token_comm = None
    try:
        out = mlp(ln, residual)
    finally:
        mlp.token_comm = comm
        store.pop_all_aux_loss(), store.pop_all_z_loss()
        for t in kept_aux:
            store.push_aux_loss(t)
        for t in kept_z:
            store.push_z_loss(t)
    return out


def is_hf_bloom(module: nn.Module) -> bool:
    """A 🤗 transformers ``BloomForCausalLM`` (the model the reference's README wraps)?"""
    cls = type(module)
    return cls.__name__ == "BloomForCausalLM" and cls.__module__.startswith("transformers.")


def hf_bloom_fast_path_blocker(hf_model) -> Optional[str]:
    """Why this 🤗 Bloom cannot run on the fused path (None: it can)."""
    c = hf_model.config
    if getattr(c, "apply_residual_connection_post_layernorm", False):
        return "apply_residual_connection_post_layernorm"
    if hf_model.lm_head.weight is not hf_model.transformer.word_embeddings.weight:
        return "untied lm_head"
    if c.hidden_size % c.n_head != 0:
        return "hidden_size not divisible by n_head"
    return None


def convert_hf_bloom_(hf_model) -> "BloomForCausalLM":
    """Turn a 🤗 ``BloomForCausalLM`` into this module's ``BloomForCausalLM`` IN PLACE: the same Python objects, the
    same ``nn.Parameter``s under the same names (optimizers, state dicts and checkpoints written from either side keep
    working) — only the container classes change, so that ``forward`` runs the fused sub-layer kernels (flash ALiBi
    attention, GEMMs with fused epilogues, fused lm_head + cross entropy) and ``TensorParallel`` can take the
    sequence-parallel path with the fused all-gather->GEMM / GEMM->reduce-scatter kernels.

    This is what ``TensorParallel(hf_bloom, ctx).parallelize()`` does for the reference's canonical input
    (reference README.md:21-69, examples/hybrid_parallelism.py:22-37)."""
    why = hf_bloom_fast_path_blocker(hf_model)
    if why is not None:
        raise ValueError(f"this Bloom cannot use the fused path: {why}")
    cfg = BloomConfig.from_hf(hf_model.config)
    cfg.tie_word_embeddings = True
    hf_config = hf_model.config
    t = hf_model.transformer
    def is_hf(mod, name):
        return type(mod).__name__ == name and type(mod).__module__.startswith("transformers.")

    for block in t.h:
        attn = block.self_attention
        attn._modules.pop("attention_dropout", None)
        attn.__class__ = BloomAttention
        attn.hidden_size, attn.num_heads, attn.head_dim = cfg.hidden_size, cfg.n_head, cfg.hidden_size // cfg.n_head
        attn.use_alibi = True
        attn._slopes_cache = {}
        # the block's MLP, or — when ExpertParallel already replaced it by an ExpertLayer — the experts inside it
        # (the ``mlp(layernorm_output, residual)`` contract is the same for both classes)
        for mlp in [m for m in block.modules() if is_hf(m, "BloomMLP")]:
            mlp._modules.pop("gelu_impl", None)
            mlp.__class__ = BloomMLP
        block.__class__ = BloomBlock
        block.eps = cfg.layer_norm_epsilon
        block.hidden_dropout = float(cfg.hidden_dropout)
        block.attention_dropout = float(cfg.attention_dropout)
        block.tp = None
    t.__class__ = BloomModel
    t.config = cfg
    hf_model.__class__ = BloomForCausalLM
    hf_model.config = cfg
    hf_model.hf_config = hf_config          # what the user built the model from (save / export helpers can read it)
    hf_model.tp = None
    hf_model.vocab_start = 0
    hf_model.lm_head.weight._pg_grad_contribs = 2   # tied table: lm_head wgrad + embedding backward
    return hf_model
