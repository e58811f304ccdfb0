"""GPT-2 on the same sm_90a sub-layer kernels as Bloom — the second model family of the reference's tests
(tests/nn/pipeline_parallel/test_partitioner.py runs its partitioner on 🤗 ``gpt2``).

A GPT-2 block is a Bloom block without ALiBi: pre-LayerNorm, fused QKV, causal softmax(QK^T/sqrt(D))V, output
projection + residual, LayerNorm, 4h MLP with the tanh GELU (🤗 ``gelu_new`` and Bloom's GELU are the same formula),
residual.  So :class:`GPT2LMHeadModel` *is* the fast ``BloomForCausalLM`` with three switches in its config — learned
position embeddings instead of ALiBi (the flash kernel runs with zero slopes), no LayerNorm after the embedding — and
inherits everything built on top of it: the sequence-parallel TensorParallel path, pipeline stages, ExpertParallel,
DataParallel / ZeRO-1, checkpoints.

Module names follow the Bloom tree (``transformer.h.N.self_attention.query_key_value`` ...); 🤗 GPT-2 checkpoints are
converted by :meth:`GPT2LMHeadModel.from_hf` (``Conv1D`` weights are transposed, and the fused QKV projection is
re-ordered from 🤗's ``[q | k | v]`` column blocks to the per-head ``(head, {q,k,v}, dim)`` layout the attention kernel
reads).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM


@dataclass
class GPT2Config(BloomConfig):
    vocab_size: int = 50257
    hidden_size: int = 768
    n_layer: int = 12
    n_head: int = 12
    n_positions: int = 1024
    position_embedding: str = "learned"
    embedding_layernorm: bool = False

    @classmethod
    def from_hf(cls, hf_config) -> "GPT2Config":
        assert getattr(hf_config, "activation_function", "gelu_new") == "gelu_new"
        assert not getattr(hf_config, "scale_attn_by_inverse_layer_idx", False)
        return cls(vocab_size=hf_config.vocab_size, hidden_size=hf_config.n_embd, n_layer=hf_config.n_layer,
                   n_head=hf_config.n_head, n_positions=hf_config.n_positions,
                   layer_norm_epsilon=hf_config.layer_norm_epsilon, initializer_range=hf_config.initializer_range)

    @classmethod
    def gpt2(cls):          # 124M
        return cls()

    @classmethod
    def gpt2_medium(cls):   # 355M
        return cls(hidden_size=1024, n_layer=24, n_head=16)

    @classmethod
    def gpt2_large(cls):    # 774M
        return cls(hidden_size=1280, n_layer=36, n_head=20)

    @classmethod
    def gpt2_xl(cls):       # 1.5B
        return cls(hidden_size=1600, n_layer=48, n_head=25)

    @classmethod
    def gpt2_tiny(cls):
        return cls(vocab_size=1024, hidden_size=128, n_layer=4, n_head=8, n_positions=128)


def _interleave_qkv(w: torch.Tensor, n_head: int) -> torch.Tensor:
    """Rows ``[q(all heads) | k | v]`` -> rows ``(head, {q,k,v}, dim)``; works for the ``[3h, h]`` weight and the ``[3h]`` bias."""
    three_h = w.shape[0]
    d = three_h // (3 * n_head)
    rest = w.shape[1:]
    return w.reshape(3, n_head, d, *rest).transpose(0, 1).reshape(three_h, *rest).contiguous()


def _deinterleave_qkv(w: torch.Tensor, n_head: int) -> torch.Tensor:
    three_h = w.shape[0]
    d = three_h // (3 * n_head)
    rest = w.shape[1:]
    return w.reshape(n_head, 3, d, *rest).transpose(0, 1).reshape(three_h, *rest).contiguous()


class GPT2LMHeadModel(BloomForCausalLM):
    def __init__(self, config: GPT2Config):
        assert config.position_embedding == "learned" and not config.embedding_layernorm
        super().__init__(config)

    # ------------------------------------------------------------------ 🤗 interop
    @staticmethod
    def convert_hf_state_dict(hf_state: dict, n_head: int) -> dict:
        """🤗 ``GPT2LMHeadModel.state_dict()`` -> this model's parameter names and layouts."""
        out = {}
        for name, t in hf_state.items():
            if name.endswith(".attn.bias") or name.endswith(".attn.masked_bias") or name == "lm_head.weight":
                continue  # causal-mask buffers; the head is tied to the embedding
            if name == "transformer.wte.weight":
                out["transformer.word_embeddings.weight"] = t
            elif name == "transformer.wpe.weight":
                out["transformer.position_embeddings.weight"] = t
            elif name.startswith("transformer.ln_f."):
                out[name] = t
            elif name.startswith("transformer.h."):
                _, _, idx, rest = name.split(".", 3)
                pre = f"transformer.h.{idx}."
                kind = rest.rsplit(".", 1)[1]           # weight | bias
                conv = (lambda x: x.t().contiguous()) if kind == "weight" else (lambda x: x)
                if rest.startswith("ln_1."):
                    out[pre + "input_layernorm." + kind] = t
                elif rest.startswith("ln_2."):
                    out[pre + "post_attention_layernorm." + kind] = t
                elif rest.startswith("attn.c_attn."):
                    out[pre + "self_attention.query_key_value." + kind] = _interleave_qkv(conv(t), n_head)
                elif rest.startswith("attn.c_proj."):
                    out[pre + "self_attention.dense." + kind] = conv(t)
                elif rest.startswith("mlp.c_fc."):
                    out[pre + "mlp.dense_h_to_4h." + kind] = conv(t)
                elif rest.startswith("mlp.c_proj."):
                    out[pre + "mlp.dense_4h_to_h." + kind] = conv(t)
                else:
                    raise KeyError(name)
            else:
                raise KeyError(name)
        return out

    @classmethod
    def from_hf(cls, hf_model) -> "GPT2LMHeadModel":
        config = GPT2Config.from_hf(hf_model.config)
        model = cls(config)
        state = cls.convert_hf_state_dict(hf_model.state_dict(), config.n_head)
        state["lm_head.weight"] = state["transformer.word_embeddings.weight"]
        model.load_state_dict(state)
        return model.to(next(hf_model.parameters()).dtype)

    def to_hf(self):
        """A 🤗 ``transformers.GPT2LMHeadModel`` with this model's weights (unsharded model; ``to_hf_state_dict`` undoes the
        weight transposes and the per-head QKV interleaving)."""
        from transformers import GPT2Config as HFConfig
        from transformers import GPT2LMHeadModel as HFGPT2

        if self.tp is not None or getattr(self, "_pg_pipeline_engine", None) is not None:
            raise ValueError("to_hf() needs the unsharded model: deparallelize() first (or consolidate the checkpoint)")
        c = self.config
        hf = HFGPT2(HFConfig(vocab_size=c.vocab_size, n_embd=c.hidden_size, n_layer=c.n_layer, n_head=c.n_head,
                             n_positions=c.n_positions, layer_norm_epsilon=c.layer_norm_epsilon,
                             initializer_range=c.initializer_range, activation_function="gelu_new",
                             resid_pdrop=c.hidden_dropout, embd_pdrop=c.hidden_dropout, attn_pdrop=c.attention_dropout))
        hf = hf.to(next(self.parameters()).dtype)
        missing, unexpected = hf.load_state_dict(self.to_hf_state_dict(), strict=False)
        assert not unexpected and all(k.endswith((".attn.bias", ".attn.masked_bias")) for k in missing), (missing, unexpected)
        hf.tie_weights()
        return hf

    def save_hf_pretrained(self, path: str, **kwargs) -> None:
        self.to_hf().save_pretrained(path, **kwargs)

    def to_hf_state_dict(self) -> dict:
        """The inverse of :meth:`convert_hf_state_dict` (unsharded model)."""
        n_head = self.config.n_head
        out = {}
        for name, t in self.state_dict().items():
            t = t.detach()
            if name == "lm_head.weight":
                out[name] = t
            elif name == "transformer.word_embeddings.weight":
                out["transformer.wte.weight"] = t
            elif name == "transformer.position_embeddings.weight":
                out["transformer.wpe.weight"] = t
            elif name.startswith("transformer.ln_f."):
                out[name] = t
            else:
                _, _, idx, rest = name.split(".", 3)
                pre = f"transformer.h.{idx}."
                kind = rest.rsplit(".", 1)[1]
                conv = (lambda x: x.t().contiguous()) if kind == "weight" else (lambda x: x)
                table = {"input_layernorm": "ln_1", "post_attention_layernorm": "ln_2", "self_attention.dense": "attn.c_proj",
                         "mlp.dense_h_to_4h": "mlp.c_fc", "mlp.dense_4h_to_h": "mlp.c_proj"}
                mod = rest.rsplit(".", 1)[0]
                if mod == "self_attention.query_key_value":
                    out[pre + "attn.c_attn." + kind] = conv(_deinterleave_qkv(t, n_head))
                elif mod in ("input_layernorm", "post_attention_layernorm"):
                    out[pre + table[mod] + "." + kind] = t
                else:
                    out[pre + table[mod] + "." + kind] = conv(t)
        return out
