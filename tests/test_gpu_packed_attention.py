"""Packed sequences on the GPU: the document-masked flash kernels (``seg_start``) against the fp32 reference, the
one-document case against the unmasked kernels, and a packed bf16 Bloom against per-document runs and under TP2."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _positions(lengths):
    return torch.cat([torch.arange(n) for n in lengths])


def _seg(layouts):
    from pipegoose_b200.ops.attention import seg_start_from_position_ids

    return seg_start_from_position_ids(torch.stack([_positions(l) for l in layouts]).cuda())


# per batch row: document lengths
LAYOUTS = {
    "blocks128": [[256, 384, 128, 256]],
    "blocks64": [[64, 192, 320, 64, 384], [448, 64, 512]],
    "inside": [[1, 37, 1, 1, 200, 90, 129, 565]],
    "ragged1000": [[300, 1, 199, 500], [1000]],
    "mixed1000": [[13, 115, 1, 871], [640, 360]],
}


@pytest.mark.parametrize("D,H", [(64, 4), (128, 2), (80, 2)])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_packed_attention_matches_reference(name, D, H):
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_attention, alibi_attention_reference

    layouts = LAYOUTS[name]
    B, S = len(layouts), sum(layouts[0])
    seg = _seg(layouts)
    torch.manual_seed(7)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    qkv_g = qkv.clone().requires_grad_(True)
    out = alibi_attention(qkv_g, slopes, B, S, H, D, seg_start=seg)     # D = 80: the zero-padded D = 128 kernel
    ref_in = qkv.float().requires_grad_(True)
    ref = alibi_attention_reference(ref_in, slopes, B, S, H, D, seg_start=seg)
    assert torch.isfinite(out).all()
    assert _rel(out, ref) < 2e-2
    dout = torch.randn_like(out)
    out.backward(dout)
    ref.backward(dout.float())
    assert torch.isfinite(qkv_g.grad).all()
    g, r = qkv_g.grad.view(B * S, H, 3, D).float(), ref_in.grad.view(B * S, H, 3, D)
    for i, part in enumerate("qkv"):
        assert _rel(g[:, :, i], r[:, :, i]) < 3e-2, part


@pytest.mark.parametrize("D,S", [(64, 1024), (128, 1000)])
def test_one_document_seg_path_is_bitwise_the_plain_kernel(D, S):
    from pipegoose_b200 import ops
    from pipegoose_b200.ops import kernels as K

    n = ops.native()
    B, H = 2, 4
    torch.manual_seed(3)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    seg = torch.zeros(B * S, dtype=torch.int32, device="cuda")
    res = {}
    for key, s in (("plain", None), ("seg", seg)):
        out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device="cuda")
        lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
        n.attention_fwd(qkv, slopes, out, lse, B, S, H, D, 0.0, s)
        dout = torch.randn(out.shape, dtype=out.dtype, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        dqkv = torch.empty_like(qkv)
        n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D, 0.0, s)
        res[key] = (out, lse, dqkv.view(B * S, H, 3, D))
    (o0, l0, g0), (o1, l1, g1) = res["plain"], res["seg"]
    assert torch.equal(o0, o1) and torch.equal(l0, l1)
    assert torch.equal(g0[:, :, 1], g1[:, :, 1]) and torch.equal(g0[:, :, 2], g1[:, :, 2])    # dK, dV
    assert _rel(g1[:, :, 0], g0[:, :, 0]) < 1e-2                                              # dQ: atomics


def test_seg_start_is_validated():
    from pipegoose_b200 import ops
    from pipegoose_b200.ops import kernels as K

    n = ops.native()
    B, S, H, D = 1, 256, 2, 64
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    for bad in (torch.zeros(S, dtype=torch.int64, device="cuda"), torch.zeros(S - 1, dtype=torch.int32, device="cuda"),
                torch.zeros(S, dtype=torch.int32)):
        with pytest.raises(RuntimeError, match="seg_start"):
            n.attention_fwd(qkv, slopes, out, lse, B, S, H, D, 0.0, bad)


def test_sdpa_fallback_masks_documents():
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_attention, alibi_attention_reference

    layouts = [[40, 1, 87, 128], [256]]
    B, S, H, D = 2, 256, 2, 160        # wider than the kernel's widest tile
    seg = _seg(layouts)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    out = alibi_attention(qkv, slopes, B, S, H, D, seg_start=seg)
    assert _rel(out, alibi_attention_reference(qkv, slopes, B, S, H, D, seg_start=seg)) < 2e-2


MODEL_LAYOUTS = [[100, 156, 256], [1, 63, 200, 248]]


def _cfg():
    from pipegoose_b200.models.bloom import BloomConfig

    return BloomConfig(vocab_size=4096, hidden_size=256, n_layer=2, n_head=4)


def test_packed_bf16_bloom_matches_per_document_runs():
    from pipegoose_b200.models.bloom import BloomForCausalLM

    torch.manual_seed(0)
    model = BloomForCausalLM(_cfg()).to(torch.bfloat16).cuda()
    solo = copy.deepcopy(model)
    B, S = len(MODEL_LAYOUTS), 512
    ids = torch.randint(0, 4096, (B, S), device="cuda")
    P = torch.stack([_positions(l) for l in MODEL_LAYOUTS]).cuda()
    loss = model(ids, labels=ids, position_ids=P).loss
    loss.backward()
    n_targets = sum(n - 1 for l in MODEL_LAYOUTS for n in l)
    total = 0.0
    for b, lengths in enumerate(MODEL_LAYOUTS):
        s0 = 0
        for n in lengths:
            if n > 1:
                doc = ids[b:b + 1, s0:s0 + n]
                part = solo(doc, labels=doc).loss * ((n - 1) / n_targets)
                part.backward()
                total += part.item()
            s0 += n
    assert abs(loss.item() - total) < 2e-2, (loss.item(), total)
    grads = dict(solo.named_parameters())
    for name, p in model.named_parameters():
        g, r = p.grad.float(), grads[name].grad.float()
        assert torch.isfinite(g).all(), name
        assert (g - r).norm().item() <= 5e-2 * r.norm().item() + 1e-6, name


def run_tp_packed(rank, world_size, port, state, ids, P, ref_loss, ref_gnorm):
    import torch.distributed as dist

    from pipegoose_b200.models.bloom import BloomForCausalLM
    from pipegoose_b200.nn import TensorParallel
    from pipegoose_b200.testing.utils import init_parallel_context

    ctx = init_parallel_context(rank, world_size, port, world_size, 1, 1, backend="nccl")
    model = BloomForCausalLM(_cfg())
    model.load_state_dict(state)
    model = TensorParallel(model.to(torch.bfloat16), ctx).parallelize()
    model.to("cuda")
    loss = model(ids.cuda(), labels=ids.cuda(), position_ids=P.cuda()).loss
    loss.backward()
    assert abs(loss.item() - ref_loss) < 3e-2, (loss.item(), ref_loss)
    sq = torch.zeros((), device="cuda")
    for n, p in model.named_parameters():
        g = p.grad.float()
        sq += g.pow(2).sum() if (hasattr(p, "parallel_metadata") and not getattr(p, "tp_partial_grad", False)) \
            else g.pow(2).sum() / world_size
    dist.all_reduce(sq)
    assert abs(sq.sqrt().item() - ref_gnorm) / ref_gnorm < 5e-2, (sq.sqrt().item(), ref_gnorm)
    ctx.destroy()


def test_tp2_packed_bloom_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pipegoose_b200.models.bloom import BloomForCausalLM
    from pipegoose_b200.testing.utils import spawn

    torch.manual_seed(0)
    ref = BloomForCausalLM(_cfg())
    state = copy.deepcopy(ref.state_dict())
    ids = torch.randint(0, 4096, (2, 512))
    P = torch.stack([_positions(l) for l in MODEL_LAYOUTS])
    model = copy.deepcopy(ref).to(torch.bfloat16).cuda()
    loss = model(ids.cuda(), labels=ids.cuda(), position_ids=P.cuda()).loss
    loss.backward()
    gnorm = torch.sqrt(sum(p.grad.float().pow(2).sum() for p in model.parameters())).item()
    spawn(run_tp_packed, world_size=2, state=state, ids=ids, P=P, ref_loss=loss.item(), ref_gnorm=gnorm)
