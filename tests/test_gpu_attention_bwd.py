"""Flash-attention backward against the fp32 reference where the model tests do not reach: lengths off the 64-query and
128-key grids (padded statistics rows, clipped dQ edge tiles), grids of several waves, short uneven documents, a dQ
workspace that held NaN before the call, and calls in a row on one stream."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _check_grads(B, S, H, D, seg=None, seed=7):
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_attention, alibi_attention_reference

    torch.manual_seed(seed)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    qkv_g = qkv.clone().requires_grad_(True)
    out = alibi_attention(qkv_g, slopes, B, S, H, D, seg_start=seg)
    ref_in = qkv.float().requires_grad_(True)
    ref = alibi_attention_reference(ref_in, slopes, B, S, H, D, seg_start=seg)
    dout = torch.randn_like(out)
    out.backward(dout)
    ref.backward(dout.float())
    assert torch.isfinite(qkv_g.grad).all()
    g, r = qkv_g.grad.view(B * S, H, 3, D).float(), ref_in.grad.view(B * S, H, 3, D)
    for i, name in enumerate("qkv"):
        assert _rel(g[:, :, i], r[:, :, i]) < 3e-2, name


# S = 1000 / 1090: the last query block is partial (stats rows padded to 64, dQ tiles clipped at S, which is also where
# the next sequence's rows begin); B * H * key blocks of 1024 and 288 CTAs: several waves on 132 SMs
@pytest.mark.parametrize("D,H,S,B", [(64, 4, 1000, 2), (64, 4, 1090, 2), (128, 2, 1000, 1), (128, 2, 1090, 2),
                                     (64, 16, 1024, 8), (128, 8, 1090, 4)])
def test_backward_matches_reference(D, H, S, B):
    _check_grads(B, S, H, D)


@pytest.mark.parametrize("D,H", [(64, 4), (128, 2)])
def test_backward_short_uneven_documents(D, H):
    from pipegoose_b200.ops.attention import seg_start_from_position_ids

    layouts = [[3, 61, 1, 130, 7, 500, 388], [1090], [64, 1, 1, 960, 64]]
    pos = torch.stack([torch.cat([torch.arange(n) for n in row]) for row in layouts]).cuda()
    _check_grads(len(layouts), 1090, H, D, seg=seg_start_from_position_ids(pos))


def _native_bwd(n, qkv, slopes, out, lse, dout, B, S, H, D):
    dqkv = torch.empty_like(qkv)
    n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D)
    return dqkv.view(B * S, H, 3, D)


@pytest.mark.parametrize("D,S", [(64, 1090), (128, 1000)])
def test_backward_workspaces_start_dirty_and_nothing_carries_over(D, S):
    """The fp32 dQ accumulator and the statistics are allocated uninitialised by every call: fill allocator blocks of
    their sizes with NaN and free them first, and run calls with other inputs in between on the same stream."""
    from pipegoose_b200 import ops
    from pipegoose_b200.ops import kernels as K

    n = ops.native()
    B, H = 2, 4
    torch.manual_seed(11)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    n.attention_fwd(qkv, slopes, out, lse, B, S, H, D)
    dout = torch.randn_like(out)
    other = torch.randn_like(out) * 100.0
    torch.cuda.synchronize()

    first = _native_bwd(n, qkv, slopes, out, lse, dout, B, S, H, D)
    s_pad = (S + 63) // 64 * 64
    for numel in (B * S * H * D, B * H * s_pad * 2):
        junk = torch.full((numel,), float("nan"), dtype=torch.float32, device="cuda")
        del junk
    dirty = _native_bwd(n, qkv, slopes, out, lse, dout, B, S, H, D)
    _native_bwd(n, qkv, slopes, out, lse, other, B, S, H, D)
    again = _native_bwd(n, qkv, slopes, out, lse, dout, B, S, H, D)
    torch.cuda.synchronize()
    for g in (dirty, again):
        assert torch.isfinite(g).all()
        # dK, dV: registers only, bitwise repeatable; dQ: fp32 sums whose order across CTAs varies
        assert torch.equal(g[:, :, 1], first[:, :, 1]) and torch.equal(g[:, :, 2], first[:, :, 2])
        assert _rel(g[:, :, 0], first[:, :, 0]) < 1e-2
