"""Head sizes without a native tile shape (bloom-3b: D=80) on the wgmma flash kernel: zero-padded to D=128 with the
softmax scale of the true width (ops/attention.py::_AlibiAttentionPadded).  Collected last on purpose."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6)).item()


@pytest.mark.parametrize("D,H,S,B", [(80, 4, 512, 2), (40, 4, 256, 1)])
def test_padded_head_attention_matches_reference(D, H, S, B):
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import alibi_attention, alibi_attention_reference, _AlibiAttentionPadded

    torch.manual_seed(7)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    qkv_g = qkv.clone().requires_grad_(True)
    out = alibi_attention(qkv_g, slopes, B, S, H, D)
    assert out.grad_fn is not None and isinstance(out.grad_fn, _AlibiAttentionPadded._backward_cls)
    ref_in = qkv.float().requires_grad_(True)
    ref = alibi_attention_reference(ref_in, slopes, B, S, H, D)
    assert _rel(out, ref) < 2e-2
    dout = torch.randn_like(out)
    out.backward(dout)
    ref.backward(dout.float())
    g, r = qkv_g.grad.view(B * S, H, 3, D).float(), ref_in.grad.view(B * S, H, 3, D)
    for i, name in enumerate("qkv"):
        assert _rel(g[:, :, i], r[:, :, i]) < 3e-2, name
