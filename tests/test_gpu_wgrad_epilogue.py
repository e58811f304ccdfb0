"""The wgrad GEMM's fp32 TMA epilogue and its fused bias gradient against float64 references.

``kernels.gemm_tn(dy, x, accum_into=main_grad, bias_grad=bias_main_grad)`` computes ``main_grad (+)= dyᵀ · x`` and
``bias_main_grad += dy.sum(0)`` in one kernel: warps 2 and 3 of the producer warpgroup sum the dy stages the main loop
already loads.  A tile sums only the k-blocks with ``kb % n_tiles == n_blk``, so every k-block of an M block is summed
once whatever the tile width and the split; an M block's sums go in with one atomic add per column and work item.

Bounds:
- weight gradient: bf16 x bf16 products are exact in fp32, so only the order of the fp32 sums differs from the
  reference; ``max|got - want| <= 1e-4 * max|want|`` as in ``test_gpu_gemm_fp32.py``;
- bias gradient, per element: recursive fp32 summation of Kc terms, then a few partial sums and the old value:
  ``|got - want| <= (Kc + 64) * 2^-24 * (sum_k |dy[k, m]| + |b0[m]|)``.  Dropping or doubling one 64-row k-block
  moves a column sum by about 8 (the sum of 64 unit normals), far above that bound at these sizes.

The CPU tests check which layers take the fused path: the bias of a row-parallel layer under tensor parallelism sums
only the local token shard while its wgrad reads every rank's tokens, so it keeps the separate column sum.
"""
import types

import pytest
import torch

EPI_ACCUM = 16
SENTINEL = -1.25e30
TOL = 1e-4
U32 = 2.0 ** -24

# (M = dy columns = weight rows, N = x columns); M edges below 64 / 128 and N edges below every tile width
SHAPES = [(1024, 1024), (3072, 1024), (264, 200), (328, 136), (8, 64)]
CONFIGS = [(None, 0), (1, 64), (2, 128), (3, 192), (8, 256), (1, 256), (4, 64)]  # (k_splits, block_n)


def _C():
    from pipegoose_b200 import ops

    return ops.native()


def _operands(M, N, Kc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(Kc, M, device="cuda", dtype=torch.bfloat16, generator=g)
    x = torch.randn(Kc, N, device="cuda", dtype=torch.bfloat16, generator=g)
    return dy, x


def _run(dy, x, out, accumulate, bias_grad, k_splits, block_n, max_ctas=0):
    ag = {} if k_splits is None else {"k_splits": k_splits}
    _C().gemm(dy, x, out, True, True, None, None, None, EPI_ACCUM if accumulate else 0, block_n, max_ctas, ag=ag,
              bias_grad=bias_grad)


def _check_bias(got, dy, b0, what):
    want = b0.double() + dy.double().sum(0)
    bound = (dy.shape[0] + 64) * U32 * (dy.double().abs().sum(0) + b0.double().abs())
    err = (got.double() - want).abs()
    worst = (err / bound).max().item()
    assert torch.isfinite(got).all() and worst <= 1.0, f"{what}: bias error {worst:.2f} x its bound"


def _check_weight(buf, M, N, expect, what):
    got = buf[:M, :N]
    assert bool((buf[M:] == SENTINEL).all() and (buf[:M, N:] == SENTINEL).all()), f"{what}: wrote outside [M, N]"
    assert torch.isfinite(got).all(), f"{what}: non-finite elements (an element was not written)"
    err = (got.double() - expect).abs().max().item()
    scale = expect.abs().max().item()
    assert err <= TOL * scale, f"{what}: weight error {err / scale:.2e} of max|want|"


@pytest.mark.gpu
@pytest.mark.parametrize("Kc", [1000, 4104, 8192])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_wgrad_with_bias_sum(shape, Kc):
    """Every tile width and forced split count, overwriting and accumulating the weight gradient, into a fresh (zero)
    and an already-filled bias gradient."""
    M, N = shape
    seed = 1000 * SHAPES.index(shape) + Kc
    dy, x = _operands(M, N, Kc, seed)
    want = dy.double().t() @ x.double()
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    w0 = torch.randn(M, N, device="cuda", dtype=torch.float32, generator=g)
    b_full = torch.randn(M, device="cuda", dtype=torch.float32, generator=g)
    for i, (k_splits, block_n) in enumerate(CONFIGS):
        accumulate = i % 2 == 1
        for b0 in (torch.zeros_like(b_full), b_full):
            buf = torch.full((M + 64, N + 8), SENTINEL, device="cuda", dtype=torch.float32)
            out = buf[:M, :N]
            if accumulate:
                out.copy_(w0)
            else:
                out.fill_(float("nan"))
            bias = b0.clone()
            _run(dy, x, out, accumulate, bias, k_splits, block_n)
            what = f"[{M}x{N}] Kc={Kc} k_splits={k_splits} block_n={block_n} accumulate={accumulate}"
            _check_weight(buf, M, N, want + w0.double() if accumulate else want, what)
            _check_bias(bias, dy, b0, what)


@pytest.mark.gpu
@pytest.mark.parametrize("k_splits", [None, 3])
def test_wgrad_bias_sum_few_ctas(k_splits):
    """4 CTAs: each walks many tiles and splits, and sums the bias over k-blocks of several M blocks."""
    M, N, Kc = 2048, 1024, 4104
    dy, x = _operands(M, N, Kc, seed=5)
    buf = torch.full((M + 64, N + 8), SENTINEL, device="cuda", dtype=torch.float32)
    out = buf[:M, :N]
    out.fill_(float("nan"))
    bias = torch.zeros(M, device="cuda", dtype=torch.float32)
    _run(dy, x, out, False, bias, k_splits, 128, max_ctas=4)
    what = f"few CTAs k_splits={k_splits}"
    _check_weight(buf, M, N, dy.double().t() @ x.double(), what)
    _check_bias(bias, dy, torch.zeros_like(bias), what)


@pytest.mark.gpu
def test_wgrad_bias_refusals():
    """The bias sum reads the A operand of a wgrad: other layouts and malformed buffers are refused."""
    dy, x = _operands(256, 128, 512, seed=9)
    out = torch.zeros(256, 128, device="cuda", dtype=torch.float32)
    with pytest.raises(RuntimeError, match="bias_grad"):
        _C().gemm(dy.t().contiguous(), x.t().contiguous(), out, False, False, None, None, None, 0,
                  bias_grad=torch.zeros(256, device="cuda", dtype=torch.float32))
    for bad in (torch.zeros(255, device="cuda", dtype=torch.float32),
                torch.zeros(256, device="cuda", dtype=torch.bfloat16),
                torch.zeros(512, device="cuda", dtype=torch.float32)[::2]):
        with pytest.raises(RuntimeError, match="bias_grad"):
            _run(dy, x, out, False, bad, None, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("fresh", [True, False])
def test_wgrad_bgrad_main_grads(fresh):
    """``functional._wgrad_bgrad`` on parameters with main grads: a fresh bias main grad (stale values from the last
    step) is cleared first, a filled one is accumulated into, exactly as the separate column sum does."""
    from pipegoose_b200.ops import functional as F

    M, N, Kc = 1024, 4096, 8192
    dy, x = _operands(M, N, Kc, seed=11)
    w = torch.nn.Parameter(torch.zeros(M, N, device="cuda", dtype=torch.bfloat16))
    b = torch.nn.Parameter(torch.zeros(M, device="cuda", dtype=torch.bfloat16))
    g = torch.Generator(device="cuda").manual_seed(12)
    w.main_grad = torch.randn(M, N, device="cuda", dtype=torch.float32, generator=g)
    b.main_grad = torch.randn(M, device="cuda", dtype=torch.float32, generator=g)
    w0, b0 = w.main_grad.clone(), b.main_grad.clone()
    w._mg_fresh = b._mg_fresh = fresh
    assert F._wgrad_bgrad(dy, x, w, b) == (None, None)
    want_w = dy.double().t() @ x.double() + (0 if fresh else w0.double())
    _check_weight(torch.nn.functional.pad(w.main_grad, (0, 8, 0, 64), value=SENTINEL), M, N, want_w, "main grads")
    _check_bias(b.main_grad, dy, torch.zeros_like(b0) if fresh else b0, "main grads")


# ---------------------------------------------------------------- which path each layer takes (CPU)
class _Recorder:
    def __init__(self, monkeypatch):
        from pipegoose_b200.ops import functional as F

        self.colsum, self.fused = 0, 0
        real_colsum, real_tn = F.K.colsum, F.K.gemm_tn

        def colsum(dy, accum_into=None):
            self.colsum += 1
            return real_colsum(dy, accum_into=accum_into)

        def gemm_tn(dy, x, accum_into=None, accumulate=True, bias_grad=None, **kw):
            self.fused += bias_grad is not None
            return real_tn(dy, x, accum_into=accum_into, accumulate=accumulate, bias_grad=bias_grad, **kw)

        monkeypatch.setattr(F.K, "colsum", colsum)
        monkeypatch.setattr(F.K, "gemm_tn", gemm_tn)


def _param(*shape, main_grad=True):
    p = torch.nn.Parameter(torch.randn(*shape))
    if main_grad:
        p.main_grad = torch.zeros(*shape)
    return p


def test_row_parallel_bias_keeps_colsum(monkeypatch):
    """Without TP the dense layer's bias gradient is summed by its wgrad; under (unfused) TP the wgrad reads the
    gathered tokens and the bias its local shard, so the column sum stays, with the local-shard result."""
    from pipegoose_b200.ops import functional as F

    torch.manual_seed(0)
    dy, a = torch.randn(16, 8), torch.randn(16, 12)
    w, b = _param(8, 12), _param(8)
    rec = _Recorder(monkeypatch)
    F._linear_residual_bwd(dy, a, w, b, None)
    assert (rec.fused, rec.colsum) == (1, 1)  # the CPU form of the fused call is a column sum
    torch.testing.assert_close(b.main_grad, dy.sum(0))
    torch.testing.assert_close(w.main_grad, dy.t() @ a)

    tp = types.SimpleNamespace(fused=False, all_gather_rows=lambda t: torch.cat([t, t]))
    w2, b2 = _param(8, 12), _param(8)
    rec2 = _Recorder(monkeypatch)
    F._linear_residual_bwd(dy, torch.cat([a, a]), w2, b2, tp)
    assert (rec2.fused, rec2.colsum) == (0, 1)
    torch.testing.assert_close(b2.main_grad, dy.sum(0))
    torch.testing.assert_close(w2.main_grad, 2 * dy.t() @ a)


def test_bias_without_main_grad_keeps_colsum(monkeypatch):
    from pipegoose_b200.ops import functional as F

    torch.manual_seed(1)
    dy, x = torch.randn(16, 8), torch.randn(16, 12)
    w, b = _param(8, 12), _param(8, main_grad=False)
    rec = _Recorder(monkeypatch)
    dw, db = F._wgrad_bgrad(dy, x, w, b)
    assert dw is None and rec.fused == 0 and rec.colsum == 1
    torch.testing.assert_close(db, dy.sum(0))
