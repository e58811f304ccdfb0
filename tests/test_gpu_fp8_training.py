"""FP8 training on one GPU: the cast kernels, the FP8 GEMM, the FP8 sub-layers and a short training run.

Casts.  ``kernels.fp8_quantize`` must give the codes, transposed codes and ``scale_inv`` of
``fp8_quantize_reference`` bit for bit.  Its column sums (the bias gradient of a dY) are recursive fp32 sums of R bf16
values: inside a 64-row tile a summation tree of depth 10 (two rows per thread, two shuffles, eight warps in order),
then one atomic add per tile into the old value, so per column, to first order,
``|got - want| <= (ceil(R / 64) + 11) * 2^-24 * (sum_r |x[r, c]| + |old[c]|)``.  Dropping a 64-row tile moves a
column sum by the sum of 64 values, far above that bound.

GEMM.  Products of two FP8 codes are exact in fp32, but FP8 wgmma accumulates them with less than fp32 precision (not
documented).  A first version of the kernel kept one tensor-core accumulator over all of K; on an H100 its error on
non-negative data reached 4.4x a model of 2^-13 lost per k32 step (1.8 % of the result at K = 1024, i.e. about 2^-10
per step), so the kernel now lets the tensor cores sum one 128-wide k-block (4 k32 steps) at a time and adds each
block's partial sums into fp32 accumulators.  The bound takes 2^-9 per k32 step (twice that measurement) inside a
block and one fp32 rounding per block, per element, with ``S = sum_k |a_k b_k| * sa * sb``:
``|acc - exact| <= E = (4 * 2^-9 + ceil(K / 128) * 2^-24) * S``.  The epilogue then adds its own roundings: the scale
product and multiply (``2^-23 |acc|``), a bf16 output (``2^-8 |out|``), ``tanh.approx`` in GELU / GELU' (``2^-10``
absolute on ``t``), and GELU / GELU' scale E by at most 1.13.  Every check also requires that dropping or doubling any
128-wide k-block of the exact product moves some element by at least 10x its bound, so the bound could not hide such
a bug (operands are non-negative, so a k-block cannot cancel out).

Sub-layers.  The FP8 attention and MLP sub-layers' output and every gradient (x, LayerNorm gamma / beta, the weights'
and biases' main grads) are compared with an fp32 unquantized reference by normalized Frobenius error.  The bound is
``1.5 * (2^-4 + 2^-3)``, a small multiple of the e4m3 and e5m2 unit roundoffs.  The residual stream passes y and dx
exactly, so ``y - x`` and ``dx - dy`` are compared.  A wrong transpose or a scale off by 2 gives an error of order 1:
the FP8 results themselves, scaled by 2 or 1/2 (and the square dense wgrad transposed), must fail the bound.  Both a
head size with its own flash tile (D = 64) and a zero-padded one (D = 80, bloom-3b) are run.

Training.  A small Bloom (h = 1024, 4 layers) memorizes a fixed batch for 100 FusedAdam steps in bf16 and in FP8 from
the same seed: both must end below half their first loss, and the FP8 final loss within 10 % of the bf16 one.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.kernels import FP8_FORMATS, fp8_quantize_reference

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
FMTS = ["e4m3", "e5m2"]


def _x(R, C, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(R, C, generator=g, device="cuda") * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------
# casts
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("shape", [(8192, 1024), (300, 136), (8, 64)])
def test_cast_is_bit_identical_to_the_reference(fmt, shape):
    R, C = shape
    x = _x(R, C, seed=R + C, scale=0.37)
    old = torch.randn(C, device="cuda")
    cs = old.clone()
    codes, codes_t, scale_inv = K.fp8_quantize(x, fmt, transpose=True, colsum_into=cs)
    torch.cuda.synchronize()
    want, want_s = fp8_quantize_reference(x.cpu(), fmt)
    assert codes.dtype == FP8_FORMATS[fmt][0] and codes_t.shape == (C, R)
    assert torch.equal(codes.cpu().view(torch.uint8), want.view(torch.uint8))
    assert torch.equal(codes_t.cpu().view(torch.uint8), want.view(torch.uint8).t().contiguous())
    assert scale_inv.cpu().view(torch.int32).item() == want_s.view(torch.int32).item()
    xd = x.double()
    ref = old.double() + xd.sum(0)
    bound = (math.ceil(R / 64) + 11) * U32 * (xd.abs().sum(0) + old.double().abs())
    err = (cs.double() - ref).abs()
    assert bool((err <= bound).all()), f"colsum: max err / bound {(err / bound).max().item():.3g}"
    if R >= 64:  # a dropped 64-row tile must exceed the bound
        assert bool(((xd[:64].sum(0)).abs() > 10 * bound).any())


@pytest.mark.parametrize("fmt", FMTS)
def test_cast_of_an_inf_gives_a_nan_scale_inv(fmt):
    x = _x(64, 64, seed=3)
    x[5, 7] = float("inf")
    _, _, scale_inv = K.fp8_quantize(x, fmt, transpose=True)
    assert torch.isnan(scale_inv).all()


def test_cast_of_zeros_and_without_optional_outputs():
    x = torch.zeros(96, 40, dtype=torch.bfloat16, device="cuda")
    codes, codes_t, scale_inv = K.fp8_quantize(x, "e4m3")
    assert codes_t is None and scale_inv.item() == 1.0
    assert bool((codes.view(torch.uint8) == 0).all())


def test_cast_refusals():
    with pytest.raises(RuntimeError, match="multiple of 8"):
        K.fp8_quantize(torch.zeros(16, 12, dtype=torch.bfloat16, device="cuda"), "e4m3")
    with pytest.raises(RuntimeError, match="contiguous"):
        K.fp8_quantize(torch.zeros(16, 32, dtype=torch.bfloat16, device="cuda")[:, :16], "e4m3")


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def _codes(x, fmt):
    c, s = fp8_quantize_reference(x.cpu(), fmt)
    return c.cuda(), s.cuda()


def _gelu(x):
    return 0.5 * x * (1 + torch.tanh(0.7978845608 * (x + 0.044715 * x ** 3)))


def _gelu_grad(x):
    t = torch.tanh(0.7978845608 * (x + 0.044715 * x ** 3))
    return 0.5 * x * (1 - t * t) * (0.7978845608 + 0.1070322243 * x * x) + 0.5 * (1 + t)


EPIS = ["bias", "bias_gelu", "bias_residual", "dgelu", "f32", "f32_accum"]
# (M, N, K, forced k_splits for the fp32 forms): M / N edges below every tile, K = 208 (one partial 128-wide k-block)
GEMM_SHAPES = [(300, 136, 208, 0), (256, 512, 1024, 0), (520, 264, 1024, 2), (64, 1024, 512, 4)]


@pytest.mark.parametrize("block_n", [64, 128])   # both FP8 tile widths; N = 136 / 264 leave partial column tiles
@pytest.mark.parametrize("a_fmt", FMTS)
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_gemm_fp8_against_float64(a_fmt, epi, shape, block_n):
    M, N, Kd, ks = shape
    kw = {"block_n": block_n}
    seed = M * 7 + N * 3 + Kd
    # non-negative operands: a dropped k-block cannot cancel out, and S equals the exact product's magnitude
    a = _x(M, Kd, seed).abs() + 0.05
    b = _x(N, Kd, seed + 1).abs() + 0.05
    ac, sa = _codes(a, a_fmt)
    bc, sb = _codes(b, "e4m3")
    ad, bd = ac.double() * sa.double(), bc.double() * sb.double()
    exact = ad @ bd.t()
    S = exact  # all products are non-negative
    E = (4 * 2.0 ** -9 + math.ceil(Kd / 128) * U32) * S + 2.0 ** -23 * exact.abs()
    bias = (_x(1, N, seed + 2).reshape(N) * 0.1)
    res = _x(M, N, seed + 3)
    z_in = _x(M, N, seed + 4)

    def out_of(acc):
        if epi == "bias":
            return acc + bias.double()
        if epi == "bias_gelu":
            return _gelu(acc + bias.double())
        if epi == "bias_residual":
            return acc + bias.double() + res.double()
        if epi == "dgelu":
            return acc * _gelu_grad(z_in.double())
        if epi == "f32":
            return acc
        return acc + old.double()

    old = torch.randn(M, N, device="cuda")
    if epi == "bias":
        got = K.gemm_fp8(ac, bc, sa, sb, bias=bias, **kw).double()
        bound = E + 2.0 ** -8 * out_of(exact).abs()
    elif epi == "bias_gelu":
        z = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        got = K.gemm_fp8(ac, bc, sa, sb, bias=bias, gelu=True, aux_out=z, **kw).double()
        pre = exact + bias.double()
        zb = E + 2.0 ** -8 * pre.abs()
        assert bool(((z.double() - pre).abs() <= zb).all()), "GELU pre-activation"
        bound = 1.13 * E + 0.5 * pre.abs() * 2.0 ** -10 + 2.0 ** -8 * _gelu(pre).abs() + 1e-6
    elif epi == "bias_residual":
        got = K.gemm_fp8(ac, bc, sa, sb, bias=bias, residual=res, **kw).double()
        bound = E + 2.0 ** -8 * out_of(exact).abs()
    elif epi == "dgelu":
        got = K.gemm_fp8(ac, bc, sa, sb, dgelu_aux=z_in, **kw).double()
        zd = z_in.double()
        dt = (zd.abs() * (0.8 + 0.11 * zd * zd) + 0.5) * 2.0 ** -10
        bound = 1.13 * E + exact.abs() * dt + 2.0 ** -8 * out_of(exact).abs() + 1e-6
    else:
        buf = old.clone()
        K.gemm_fp8(ac, bc, sa, sb, accum_into=buf, accumulate=epi == "f32_accum", k_splits=ks, **kw)
        got = buf.double()
        bound = E + 4 * U32 * out_of(exact).abs()
    want = out_of(exact)
    err = (got - want).abs()
    ratio = (err / bound).max().item()
    assert ratio <= 1.0, f"max |err| / bound = {ratio:.3g}"
    # the bound must catch a dropped or doubled 128-wide k-block
    for kb in range(0, Kd, 128):
        part = ad[:, kb:kb + 128] @ bd[:, kb:kb + 128].t()
        for mistake in (exact - part, exact + part):
            assert ((out_of(mistake) - want).abs() / bound).max().item() >= 10, f"k-block {kb // 128}"


def test_gemm_fp8_refuses_tiles_wider_than_128():
    a = torch.zeros(128, 128, device="cuda").to(torch.float8_e4m3fn)
    s = torch.ones(1, device="cuda")
    with pytest.raises(RuntimeError, match="block_n"):
        K.gemm_fp8(a, a, s, s, block_n=256)


def test_gemm_fp8_refusals():
    a = torch.zeros(64, 40, device="cuda").to(torch.float8_e4m3fn)
    s = torch.ones(1, device="cuda")
    with pytest.raises(RuntimeError, match="16"):
        K.gemm_fp8(a, a, s, s)
    b = torch.zeros(64, 64, device="cuda").to(torch.float8_e5m2)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        K.gemm_fp8(b, b, s, s)


# ------------------------------------------------------------------------------------------------------------------
# sub-layers
# ------------------------------------------------------------------------------------------------------------------
SUB_BOUND = 1.5 * (2.0 ** -4 + 2.0 ** -3)


def _rel(got, want):
    return ((got.float() - want.float()).norm() / want.float().norm()).item()


def _params(h, n_out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(n_out, h, generator=g, device="cuda") / math.sqrt(h)).to(torch.bfloat16)
    b = (torch.randn(n_out, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
    return w, b


def _with_main_grads(ts):
    out = []
    for t in ts:
        p = t.detach().clone().requires_grad_(True)
        p.main_grad = torch.zeros(t.shape, dtype=torch.float32, device="cuda")
        out.append(p)
    return out


def _ref_leaves(ts):
    return [t.detach().float().clone().requires_grad_(True) for t in ts]


def _compared(x, x0, y, xr, yr, dy, names, p, pr):
    """The sub-layer's results against the reference.  The residual stream passes y = x + ... and dx = dy + ...
    exactly, so it is taken out of both: it would dilute the FP8 error."""
    named = {"y - x": (y.detach().float() - x0.float(), yr.detach() - x0.float()),
             "dx - dy": (x.grad.float() - dy.float(), xr.grad - dy.float())}
    named.update({n: (q.main_grad, r.grad) for n, q, r in zip(names, p, pr)})
    return named


def _check(named):
    errs = {k: _rel(g, w) for k, (g, w) in named.items()}
    bad = {k: e for k, e in errs.items() if not e <= SUB_BOUND}
    assert not bad, f"normalized errors above {SUB_BOUND:.3f}: {bad} (all: {errs})"
    return errs


@pytest.mark.parametrize("h, n_head", [(1024, 16), (1280, 16)])   # D = 64 and D = 80 (zero-padded attention)
def test_attention_sublayer_fp8_against_fp32(h, n_head):
    from pipegoose_b200.ops import functional as PF
    from pipegoose_b200.ops.attention import alibi_attention_reference

    B, S = 2, 256
    D = h // n_head
    x0 = _x(B * S, h, 11)
    gamma = (1 + 0.1 * _x(1, h, 12).reshape(h)).to(torch.bfloat16)
    beta = (0.1 * _x(1, h, 13).reshape(h)).to(torch.bfloat16)
    wq, bq = _params(h, 3 * h, 14)
    wd, bdn = _params(h, h, 15)
    slopes = K.alibi_slopes(n_head, device="cuda")
    dy = _x(B * S, h, 16)
    params = [gamma, beta, wq, bq, wd, bdn]

    x = x0.clone().requires_grad_(True)
    p = _with_main_grads(params)
    y = PF.attention_sublayer_fp8(x, *p[:6], slopes, 1e-5, B, S, n_head, D)
    y.backward(dy)

    xr = x0.float().clone().requires_grad_(True)
    pr = _ref_leaves(params)
    ln = F.layer_norm(xr, (h,), pr[0], pr[1], 1e-5)
    qkv = F.linear(ln, pr[2], pr[3])
    att = alibi_attention_reference(qkv, slopes, B, S, n_head, D)
    yr = F.linear(att, pr[4], pr[5]) + xr
    yr.backward(dy.float())
    names = ["gamma", "beta", "w_qkv", "b_qkv", "w_dense", "b_dense"]
    _check(_compared(x, x0, y, xr, yr, dy, names, p, pr))
    # the bound rejects the FP8 results with a scale off by 2, and a transposed dense wgrad (a square [h, h] matrix)
    for got, want in ((y.detach().float() - x0.float(), yr.detach() - x0.float()), (p[2].main_grad, pr[2].grad),
                      (p[4].main_grad, pr[4].grad)):
        assert _rel(2 * got, want) > 3 * SUB_BOUND and _rel(0.5 * got, want) > SUB_BOUND
    assert _rel(p[4].main_grad.t(), pr[4].grad) > 3 * SUB_BOUND


def test_layernorm_mlp_fp8_against_fp32():
    from pipegoose_b200.ops import functional as PF

    M, h = 512, 1024
    x0 = _x(M, h, 21)
    gamma = (1 + 0.1 * _x(1, h, 22).reshape(h)).to(torch.bfloat16)
    beta = (0.1 * _x(1, h, 23).reshape(h)).to(torch.bfloat16)
    w1, b1 = _params(h, 4 * h, 24)
    w2, b2 = _params(4 * h, h, 25)
    dy = _x(M, h, 27)
    params = [gamma, beta, w1, b1, w2, b2]

    x = x0.clone().requires_grad_(True)
    p = _with_main_grads(params)
    y = PF.layernorm_mlp_fp8(x, *p, 1e-5)
    y.backward(dy)

    xr = x0.float().clone().requires_grad_(True)
    pr = _ref_leaves(params)
    ln = F.layer_norm(xr, (h,), pr[0], pr[1], 1e-5)
    yr = F.linear(_gelu(F.linear(ln, pr[2], pr[3])), pr[4], pr[5]) + xr
    yr.backward(dy.float())
    names = ["gamma", "beta", "w_fc1", "b_fc1", "w_fc2", "b_fc2"]
    _check(_compared(x, x0, y, xr, yr, dy, names, p, pr))
    for got, want in ((p[2].main_grad, pr[2].grad), (p[4].main_grad, pr[4].grad)):
        assert _rel(2 * got, want) > 3 * SUB_BOUND and _rel(0.5 * got, want) > SUB_BOUND


def test_attention_sublayer_fp8_refuses_head_sizes_without_a_flash_tile():
    from pipegoose_b200.ops import functional as PF

    h, n_head, D = 512, 2, 256
    x = _x(256, h, 41)
    wq, bq = _params(h, 3 * h, 42)
    wd, bdn = _params(h, h, 43)
    g = torch.ones(h, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="head size"):
        PF.attention_sublayer_fp8(x, g, g, wq, bq, wd, bdn, K.alibi_slopes(n_head, device="cuda"), 1e-5, 1, 256,
                                  n_head, D)


def test_sublayers_return_grads_without_main_grads():
    from pipegoose_b200.ops import functional as PF

    M, h = 256, 256
    x = _x(M, h, 31).requires_grad_(True)
    gamma = torch.ones(h, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    beta = torch.zeros(h, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    w1, b1 = [t.requires_grad_(True) for t in _params(h, 4 * h, 32)]
    w2, b2 = [t.requires_grad_(True) for t in _params(4 * h, h, 33)]
    PF.layernorm_mlp_fp8(x, gamma, beta, w1, b1, w2, b2, 1e-5).float().sum().backward()
    for t in (x, gamma, beta, w1, b1, w2, b2):
        assert t.grad is not None and t.grad.dtype == torch.bfloat16 and bool(torch.isfinite(t.grad).all())


# ------------------------------------------------------------------------------------------------------------------
# training
# ------------------------------------------------------------------------------------------------------------------
def _train(fp8: bool, steps: int = 100):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.optim import FusedAdam

    torch.manual_seed(0)
    cfg = BloomConfig(vocab_size=4096, hidden_size=1024, n_layer=4, n_head=16, fp8=fp8)
    model = BloomForCausalLM(cfg).to(torch.bfloat16).cuda()
    opt = FusedAdam(model.parameters(), lr=3e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (4, 256), device="cuda", generator=g)
    losses = []
    for _ in range(steps):
        loss = model(ids, labels=ids).loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    return [l.item() for l in losses]


def test_fp8_training_memorizes_like_bf16():
    bf16 = _train(False)
    fp8 = _train(True)
    print(f"bf16 first / last {bf16[0]:.4f} / {bf16[-1]:.4f}; fp8 first / last {fp8[0]:.4f} / {fp8[-1]:.4f}")
    assert all(math.isfinite(v) for v in fp8)
    assert bf16[-1] < 0.5 * bf16[0] and fp8[-1] < 0.5 * fp8[0]
    assert abs(fp8[-1] - bf16[-1]) <= 0.1 * bf16[-1]
