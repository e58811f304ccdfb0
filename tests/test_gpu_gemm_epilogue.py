"""The GEMM's TMA-store epilogue (bf16 output, one chunk, 16-byte-aligned matrices) against the general epilogue.

Both epilogues apply the same fp32 arithmetic in the same order, so every bf16 output must be bit-identical.  The
general epilogue is reached in the same process with ``num_chunks=2`` and no peers or flags: a plain GEMM visited as
two row chunks (M a multiple of 256).  Only the cross-entropy partial sums are summed in a different order."""
import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_BIAS, EPI_GELU, EPI_RESIDUAL, EPI_DGELU = 1, 2, 4, 32
FORMS = ["none", "bias", "bias_gelu_aux", "bias_residual", "dgelu"]


def _C():
    from pipegoose_b200 import ops

    return ops.native()


def _operands(M, N, K, layout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16, generator=g)
    if layout == "nt":
        b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16, generator=g)
    else:  # nn: B stored [K, N]
        b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16, generator=g)
    bias = torch.randn(N, device="cuda", dtype=torch.bfloat16, generator=g)
    # residual / GELU' input, with the outputs' leading dimension (a GELU' input must share it)
    mat = torch.randn(M, N + 8, device="cuda", dtype=torch.bfloat16, generator=g)[:, :N]
    return a, b, bias, mat


def _padded(M, N):
    """[M, N] bf16 view of a NaN-filled [M + 64, N + 8] buffer: a store past the M or N edge would show in the margin."""
    return torch.full((M + 64, N + 8), float("nan"), device="cuda", dtype=torch.bfloat16)[:M, :N]


def _margin_untouched(view):
    M, N = view.shape
    buf = torch.as_strided(view, (M + 64, N + 8), view.stride())
    return bool(torch.isnan(buf[M:]).all() and torch.isnan(buf[:, N:]).all())


def _gemm(form, a, b, layout, bias, mat, **kw):
    M, N = a.shape[0], (b.shape[0] if layout == "nt" else b.shape[1])
    out = _padded(M, N)
    aux = None
    flags = 0
    use_bias = bias if form.startswith("bias") else None
    res = mat if form == "bias_residual" else None
    if form == "bias_gelu_aux":
        flags, aux = EPI_GELU, _padded(M, N)
    elif form == "dgelu":
        flags, aux = EPI_DGELU, mat
    _C().gemm(a, b, out, False, layout == "nn", use_bias, res, aux, flags, **kw)
    assert _margin_untouched(out) and (aux is None or form == "dgelu" or _margin_untouched(aux))
    return out.clone(), (aux.clone() if form == "bias_gelu_aux" else None)


def _reference(form, a, b, layout, bias, mat):
    """fp32 (output, pre-activation) of the same GEMM and epilogue."""
    from pipegoose_b200.ops import kernels as K

    pre = a.float() @ (b.float().t() if layout == "nt" else b.float())
    if form.startswith("bias"):
        pre = pre + bias.float()
    out = {"bias_gelu_aux": lambda: K.gelu_tanh(pre), "bias_residual": lambda: pre + mat.float(),
           "dgelu": lambda: pre * K.gelu_tanh_grad(mat.float())}.get(form, lambda: pre)()
    return out, pre


def _assert_close(got, want):
    assert (got.float() - want).abs().max().item() <= 2e-2 * want.abs().max().item()


def _assert_same(new, old):
    assert torch.equal(new[0], old[0]), (new[0].float() - old[0].float()).abs().max()
    if new[1] is not None:
        assert torch.equal(new[1], old[1]), (new[1].float() - old[1].float()).abs().max()


@pytest.mark.parametrize("layout", ["nt", "nn"])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("block_n", [0, 128, 256])
def test_tma_epilogue_bit_identical_to_chunked_path(layout, form, block_n):
    a, b, bias, mat = _operands(512, 768, 320, layout, seed=11)
    new = _gemm(form, a, b, layout, bias, mat, block_n=block_n)
    old = _gemm(form, a, b, layout, bias, mat, block_n=block_n, num_chunks=2)
    _assert_same(new, old)
    want, pre = _reference(form, a, b, layout, bias, mat)
    _assert_close(new[0], want)
    if form == "bias_gelu_aux":
        _assert_close(new[1], pre)


@pytest.mark.parametrize("layout", ["nt", "nn"])
@pytest.mark.parametrize("shape", [(1000, 264, 200), (640, 328, 136)])
@pytest.mark.parametrize("block_n", [64, 128, 192, 256])
@pytest.mark.parametrize("form", FORMS)
def test_tma_epilogue_edges(layout, shape, block_n, form):
    """M and N tails (the TMA boxes are clipped: the margin around the output stays untouched) at every tile width."""
    M, N, K = shape
    a, b, bias, mat = _operands(M, N, K, layout, seed=12)
    new = _gemm(form, a, b, layout, bias, mat, block_n=block_n)
    want, pre = _reference(form, a, b, layout, bias, mat)
    _assert_close(new[0], want)
    if form == "bias_gelu_aux":
        _assert_close(new[1], pre)


@pytest.mark.parametrize("form", ["none", "bias_gelu_aux", "bias_residual", "dgelu"])
def test_tma_epilogue_many_tiles_per_cta(form):
    """4 CTAs over 256 tiles: every CTA reuses its slots and drains its stores across 64 tiles."""
    a, b, bias, mat = _operands(2048, 2048, 192, "nt", seed=13)
    new = _gemm(form, a, b, "nt", bias, mat, block_n=128, max_ctas=4)
    old = _gemm(form, a, b, "nt", bias, mat, block_n=128, max_ctas=4, num_chunks=2)
    _assert_same(new, old)


@pytest.mark.parametrize("layout", ["nt", "nn"])
@pytest.mark.parametrize("M,V,valid", [(512, 4096, 4096), (768, 2560, 2500), (256, 1000, 1000)])
def test_tma_epilogue_ce_partials(layout, M, V, valid):
    """lm_head form: logits bit-identical, per-row log-sum-exp of the partials equal up to summation order."""
    from pipegoose_b200.ops import kernels as K

    a, b, _, _ = _operands(M, V, 256, layout, seed=14)
    a, b = a * 0.5, b * 0.2
    outs = {}
    for name, kw in (("new", {}), ("old", {"num_chunks": 2})):
        part = K.ce_partials_buffer(M, V, a.device).fill_(float("nan"))
        logits = torch.empty(M, V, device="cuda", dtype=torch.bfloat16)
        _C().gemm(a, b, logits, False, layout == "nn", None, None, None, 0,
                  ag={"ce_part": part.data_ptr(), "ce_valid": valid}, **kw)
        assert not torch.isnan(part).any(), name
        lse = torch.logsumexp(part[..., 0] + torch.log(part[..., 1]), dim=1)
        outs[name] = (logits, lse)
    assert torch.equal(outs["new"][0], outs["old"][0])
    want = torch.logsumexp(outs["new"][0][:, :valid].float(), dim=1)
    assert torch.allclose(outs["new"][1], outs["old"][1], rtol=1e-6, atol=1e-5)
    assert torch.allclose(outs["new"][1], want, rtol=1e-6, atol=1e-5)


def test_misaligned_output_is_rejected():
    """Both epilogues write 16-byte groups: an output that does not start on 16 bytes is an error, not a fault."""
    a, b, _, _ = _operands(256, 128, 64, "nt", seed=15)
    buf = torch.empty(256, 136, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="16B aligned"):
        _C().gemm(a, b, buf[:, 4:132], False, False)
