"""Packed sequences: several documents in one row, described by ``position_ids`` that restart at 0 on every document.
The packed run must equal every document run on its own (attention, loss, gradients), and ``position_ids = arange``
must equal no ``position_ids`` at all."""
import copy

import numpy as np
import pytest
import torch

from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel
from pipegoose_b200.ops.attention import (alibi_attention_reference, alibi_attention_with_dropout,
                                          seg_start_from_position_ids)
from pipegoose_b200.ops.kernels import alibi_slopes
from pipegoose_b200.utils.data import TokenFileDataset, write_token_file


def _positions(lengths):
    return torch.cat([torch.arange(n) for n in lengths])


# per batch row: document lengths (each row sums to S = 24)
LAYOUTS = [[1, 5, 1, 9, 8], [24]]
LAYOUTS_B3 = [[7, 1, 16], [24], [3, 3, 3, 3, 12]]


@pytest.mark.parametrize("layouts", [LAYOUTS, LAYOUTS_B3, [[1] * 24]])
def test_reference_attention_with_seg_start_equals_per_document_runs(layouts):
    torch.manual_seed(0)
    B, S, H, D = len(layouts), 24, 4, 16
    qkv = torch.randn(B * S, H * 3 * D)
    slopes = alibi_slopes(H, device="cpu")
    P = torch.stack([_positions(l) for l in layouts])
    out = alibi_attention_reference(qkv, slopes, B, S, H, D, seg_start=seg_start_from_position_ids(P)).view(B, S, -1)
    rows = qkv.view(B, S, -1)
    for b, lengths in enumerate(layouts):
        s0 = 0
        for n in lengths:
            doc = rows[b, s0:s0 + n].reshape(n, -1)
            ref = alibi_attention_reference(doc, slopes, 1, n, H, D)
            torch.testing.assert_close(out[b, s0:s0 + n], ref, rtol=1e-5, atol=1e-5)
            s0 += n
    # one document per row: the plain causal attention
    whole = torch.zeros(B, S, dtype=torch.int32)
    assert torch.equal(alibi_attention_reference(qkv, slopes, B, S, H, D, seg_start=whole),
                       alibi_attention_reference(qkv, slopes, B, S, H, D))


def test_dropout_path_masks_documents():
    torch.manual_seed(0)
    B, S, H, D = 2, 24, 4, 16
    qkv = torch.randn(B * S, H * 3 * D)
    slopes = alibi_slopes(H, device="cpu")
    seg = seg_start_from_position_ids(torch.stack([_positions(l) for l in LAYOUTS]))
    # a vanishing dropout probability keeps every entry: the masking is what is compared
    out = alibi_attention_with_dropout(qkv, slopes, B, S, H, D, 1e-12, seg_start=seg)
    torch.testing.assert_close(out, alibi_attention_reference(qkv, slopes, B, S, H, D, seg_start=seg),
                               rtol=1e-5, atol=1e-5)


def _bloom():
    torch.manual_seed(0)
    return BloomForCausalLM(BloomConfig.bloom_tiny())


def _gpt2():
    torch.manual_seed(0)
    return GPT2LMHeadModel(GPT2Config.gpt2_tiny())


@pytest.mark.parametrize("make", [_bloom, _gpt2], ids=["bloom", "gpt2"])
@pytest.mark.parametrize("recompute", ["none", "block"])
def test_packed_loss_and_gradients_equal_per_document_runs(make, recompute):
    model = make()
    model.config.recompute = recompute
    solo = copy.deepcopy(model)
    layouts = LAYOUTS_B3
    B, S = len(layouts), 24
    ids = torch.randint(0, model.config.vocab_size, (B, S))
    P = torch.stack([_positions(l) for l in layouts])
    loss = model(ids, labels=ids, position_ids=P).loss
    loss.backward()

    n_targets = sum(n - 1 for l in layouts for n in l)
    total = torch.zeros(())
    for b, lengths in enumerate(layouts):
        s0 = 0
        for n in lengths:
            if n > 1:   # a one-token document has no target
                doc = ids[b:b + 1, s0:s0 + n]
                part = solo(doc, labels=doc).loss * ((n - 1) / n_targets)
                part.backward()
                total = total + part.detach()
            s0 += n
    torch.testing.assert_close(loss.detach(), total, rtol=1e-5, atol=1e-6)
    grads = dict(solo.named_parameters())
    for name, p in model.named_parameters():
        torch.testing.assert_close(p.grad, grads[name].grad, rtol=1e-4, atol=1e-6, msg=name)


@pytest.mark.parametrize("make", [_bloom, _gpt2], ids=["bloom", "gpt2"])
def test_arange_position_ids_are_bitwise_no_position_ids(make):
    model = make()
    other = copy.deepcopy(model)
    ids = torch.randint(0, model.config.vocab_size, (2, 24))
    P = torch.arange(24).expand(2, 24)
    a = model(ids, labels=ids)
    b = other(ids, labels=ids, position_ids=P)
    assert torch.equal(a.loss, b.loss)
    a.loss.backward()
    b.loss.backward()
    grads = dict(other.named_parameters())
    for name, p in model.named_parameters():
        assert torch.equal(p.grad, grads[name].grad), name
    with torch.no_grad():
        assert torch.equal(model(ids).logits, other(ids, position_ids=P).logits)


@pytest.mark.parametrize("bad", [
    [1, 2, 3, 4, 5, 6],       # does not start at 0
    [0, 1, 3, 4, 5, 6],       # a step of +2
    [0, 1, 2, 1, 2, 3],       # a reset to 1
    [0, 1, 2, 2, 3, 4],       # a step of 0
])
def test_malformed_position_ids_raise(bad):
    model = _bloom()
    ids = torch.randint(0, 64, (2, 6))
    P = torch.stack([torch.arange(6), torch.tensor(bad)])
    with pytest.raises(RuntimeError, match="position_ids"):
        model(ids, labels=ids, position_ids=P)


def test_position_ids_shape_and_dtype_are_checked():
    model = _bloom()
    ids = torch.randint(0, 64, (2, 6))
    with pytest.raises(ValueError, match="shape"):
        model(ids, labels=ids, position_ids=torch.arange(6)[None])
    with pytest.raises(ValueError, match="integer"):
        model(ids, labels=ids, position_ids=torch.arange(6.0).expand(2, 6))


def test_position_ids_with_a_holed_mask_raise():
    model = _bloom()
    ids = torch.randint(0, 64, (2, 6))
    P = torch.tensor([[0, 1, 2, 0, 1, 2]] * 2)
    mask = torch.ones(2, 6, dtype=torch.long)
    mask[1, 4:] = 0
    with pytest.raises(ValueError, match="attention_mask"):
        model(ids, attention_mask=mask, labels=ids, position_ids=P)
    # an all-ones mask says nothing the positions do not
    a = model(ids, attention_mask=torch.ones_like(mask), labels=ids, position_ids=P).loss
    b = model(ids, labels=ids, position_ids=P).loss
    assert torch.equal(a, b)


def test_pipeline_engines_refuse_position_ids():
    from pipegoose_b200.nn.pipeline_parallel.job_engine import JobPipelineEngine
    from pipegoose_b200.nn.pipeline_parallel.pipeline_engine import PipelineEngine

    ids = torch.zeros(2, 6, dtype=torch.long)
    P = torch.tensor([[0, 1, 2, 0, 1, 2]] * 2)
    for engine in (PipelineEngine, JobPipelineEngine):
        stub = object.__new__(engine)      # the refusal comes before the engine touches any of its state
        with pytest.raises(ValueError, match="position_ids"):
            engine.run(stub, input_ids=ids, labels=ids, position_ids=P)


def test_token_file_dataset_position_ids(tmp_path):
    path = str(tmp_path / "tokens.bin")
    eos = 1
    tokens = [5, 6, 1, 7, 1, 1, 8, 9, 10, 1, 11, 12]
    write_token_file(path, tokens)
    plain = TokenFileDataset(path, seq_len=6)
    packed = TokenFileDataset(path, seq_len=6, eos_token_id=eos)
    assert set(plain[0]) == {"input_ids"}
    assert len(plain) == len(packed) == 2
    for i in range(2):
        assert torch.equal(plain[i]["input_ids"], packed[i]["input_ids"])
        assert packed[i]["position_ids"].dtype == torch.int64
    # window 0: [5 6 1 | 7 1 | 1]; window 1: [8 9 10 1 | 11 12]
    assert packed[0]["position_ids"].tolist() == [0, 1, 2, 0, 1, 0]
    assert packed[1]["position_ids"].tolist() == [0, 1, 2, 3, 0, 1]
    # an overlapping window starts its first document at 0 wherever it begins
    strided = TokenFileDataset(path, seq_len=6, stride=1, eos_token_id=eos)
    assert strided[1]["position_ids"].tolist() == [0, 1, 0, 1, 0, 0]
    assert strided[1]["input_ids"].tolist() == [6, 1, 7, 1, 1, 8]
    # the items train as they come out of the dataset
    model = _bloom()
    batch = torch.utils.data.default_collate([packed[0], packed[1]])
    out = model(**batch, labels=batch["input_ids"])
    assert torch.isfinite(out.loss)


def test_packed_positions_match_a_python_loop():
    from pipegoose_b200.utils.data import _packed_positions

    rng = np.random.default_rng(0)
    toks = rng.integers(0, 4, size=200)
    expect, p = [], 0
    for i, t in enumerate(toks):
        if i > 0 and toks[i - 1] == 0:
            p = 0
        expect.append(p)
        p += 1
    assert _packed_positions(toks, 0).tolist() == expect
