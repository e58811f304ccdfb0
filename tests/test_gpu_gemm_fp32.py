"""The GEMM with an fp32 output (wgrad into the fp32 main gradients) against a float64 reference.

This is the TN form ``out[N, K] (+)= dyᵀ · x`` that ``kernels.gemm_tn`` runs for every weight gradient.  For fp32 outputs
``pg_gemm_bf16`` may split the contraction over several work items per tile (split-K, automatically or through the
``k_splits`` override); the partial sums are then added with ``red.global.add``, after a ``cudaMemset2DAsync`` of the
``[N, K]`` output when the call overwrites instead of accumulating.

bf16 x bf16 products are exact in fp32, so the only error is the order of the fp32 sums.  The bound
``max|got - want| <= 1e-4 * max|want|`` is far below what the smallest plausible bug does: dropping or doubling one
64-wide k-block changes the result by about ``sqrt(64 / Kc)`` relative, >= 6e-2 even at ``Kc = 16392``.  On one H100
80GB HBM3 (700 W power limit) the largest error measured over these shapes, contractions and splits was 2.1e-5 of
max|want| (at 8 x 64, Kc = 16392).

Which calls split on their own (same H100, read from a profiler trace: the kernel's tile width, its grid and whether
the memset ran): at bloom-560m's B·S = 8192 the 1024 x 1024 wgrad splits 4 ways at BN = 256 (32 tiles, 128 CTAs) and the
3072 x 1024 one splits at BN = 256 (96 tiles, 132 CTAs); 4096 x 1024 and 1024 x 4096 do not split.  The 264 x 200 and
328 x 136 tails split at BN = 64 from Kc = 4104 up; nothing splits at Kc = 1024 or below.

Every destination is an ``[N, K]`` view of an ``[N + 64, K + 8]`` buffer whose margin holds a sentinel; the margin must be
bitwise unchanged, which catches the memset, the atomics or the plain stores writing past N, past K or past a row.
An overwriting call starts from NaN, so every element it fails to write shows.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_ACCUM = 16
SENTINEL = -1.25e30
TOL = 1e-4

OUT_SHAPES = [(1024, 1024), (3072, 1024), (4096, 1024), (1024, 4096), (264, 200), (328, 136), (8, 64)]
CONTRACTIONS = [64, 640, 1000, 1024, 4104, 8192, 16392]
BLOCK_NS = [0, 64, 128, 192, 256]


def _C():
    from pipegoose_b200 import ops

    return ops.native()


def _operands(N, K, Kc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(Kc, N, device="cuda", dtype=torch.bfloat16, generator=g)
    x = torch.randn(Kc, K, device="cuda", dtype=torch.bfloat16, generator=g)
    return dy, x


def _reference(dy, x):
    return dy.double().t() @ x.double()


def _destination(N, K, fill):
    """[N, K] fp32 view (fill) of an [N + 64, K + 8] buffer whose margin holds SENTINEL."""
    buf = torch.full((N + 64, K + 8), SENTINEL, device="cuda", dtype=torch.float32)
    view = buf[:N, :K]
    if isinstance(fill, torch.Tensor):
        view.copy_(fill)
    else:
        view.fill_(fill)
    return view, buf


def _margin_intact(buf, N, K):
    return bool((buf[N:] == SENTINEL).all() and (buf[:N, K:] == SENTINEL).all())


def _gemm(dy, x, out, accumulate, k_splits=None, block_n=0, max_ctas=0):
    ag = {} if k_splits is None else {"k_splits": k_splits}
    _C().gemm(dy, x, out, True, True, None, None, None, EPI_ACCUM if accumulate else 0, block_n, max_ctas, ag=ag)


def _assert_close(got, want, what):
    assert torch.isfinite(got).all(), f"{what}: non-finite elements (an element was not written)"
    err = (got.double() - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= TOL * scale, f"{what}: max error {err:.3e} = {err / scale:.2e} of max|want| {scale:.3e}"


def _check(dy, x, want, accumulate, k_splits=None, block_n=0, max_ctas=0, seed=0):
    N, K = want.shape
    if accumulate:
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        a0 = torch.randn(N, K, device="cuda", dtype=torch.float32, generator=g)
        out, buf = _destination(N, K, a0)
        expect = a0.double() + want
    else:
        out, buf = _destination(N, K, float("nan"))
        expect = want
    _gemm(dy, x, out, accumulate, k_splits, block_n, max_ctas)
    what = f"[{N}x{K}] Kc={dy.shape[0]} accumulate={accumulate} k_splits={k_splits} block_n={block_n} max_ctas={max_ctas}"
    assert _margin_intact(buf, N, K), f"{what}: wrote outside the [N, K] view"
    _assert_close(out, expect, what)


@pytest.mark.parametrize("Kc", CONTRACTIONS)
@pytest.mark.parametrize("shape", OUT_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_fp32_gemm_splits(shape, Kc):
    """Automatic split, split forced off, 2 / 3 / 7 / 8 splits and more splits than k-blocks (clamped, no empty split),
    each overwriting and accumulating, with the tile width rotating through every BN over the matrix."""
    N, K = shape
    si, ki = OUT_SHAPES.index(shape), CONTRACTIONS.index(Kc)
    dy, x = _operands(N, K, Kc, seed=100 * si + ki)
    want = _reference(dy, x)
    num_kb = (Kc + 63) // 64
    configs = [(None, 0)] + [(s, BLOCK_NS[(j + si + ki) % len(BLOCK_NS)])
                             for j, s in enumerate([1, 2, 3, 7, 8, num_kb + 3])]
    for accumulate in (False, True):
        for k_splits, block_n in configs:
            _check(dy, x, want, accumulate, k_splits, block_n, seed=si * 7 + ki)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("k_splits", [None, 1, 3, 8])
def test_fp32_gemm_few_ctas(accumulate, k_splits):
    """4 CTAs: every CTA walks many work items, across tiles and across the splits of one tile."""
    dy, x = _operands(2048, 1024, 4104, seed=7)
    want = _reference(dy, x)
    _check(dy, x, want, accumulate, k_splits, 128 if k_splits is not None else 0, max_ctas=4)


def test_fp32_gemm_stream_order():
    """Kernels that write one buffer back to back, with no synchronisation in between, stay ordered (the GEMM is
    launched with programmatic dependent launch): an overwriting split GEMM, an accumulating split GEMM, a bf16 -> fp32
    gradient accumulation and a column sum into one row of the buffer."""
    from pipegoose_b200.ops import kernels as K_

    N, K, Kc = 1024, 1024, 8192
    dy1, x1 = _operands(N, K, Kc, seed=21)
    dy2, x2 = _operands(N, K, Kc, seed=22)
    g = torch.Generator(device="cuda").manual_seed(23)
    grad = torch.randn(N, K, device="cuda", dtype=torch.bfloat16, generator=g)
    cs = torch.randn(4096, K, device="cuda", dtype=torch.bfloat16, generator=g)
    want = _reference(dy1, x1) + _reference(dy2, x2) + grad.double()
    want[0] += cs.double().sum(0)
    buf = torch.full((N, K), float("nan"), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    _gemm(dy1, x1, buf, False, k_splits=4)
    _gemm(dy2, x2, buf, True, k_splits=3)
    K_.accumulate_grad(grad, buf)
    K_.colsum(cs, accum_into=buf[0])
    _assert_close(buf, want, "stream-ordered chain")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("rows", [8192, 8200])
@pytest.mark.parametrize("shape", [(1024, 1024), (3072, 1024), (4096, 1024), (1024, 4096)],
                         ids=lambda s: f"{s[0]}x{s[1]}")
def test_gemm_tn_main_grad(shape, rows, accumulate):
    """``kernels.gemm_tn`` into a contiguous fp32 main gradient at bloom-560m's wgrad shapes (B·S = 8192 rows, and a
    ragged 8200), as training calls it."""
    from pipegoose_b200.ops import kernels as K_

    N, K = shape
    dy, x = _operands(N, K, rows, seed=31 + rows + N)
    want = _reference(dy, x)
    g = torch.Generator(device="cuda").manual_seed(32)
    main = torch.randn(N * K, device="cuda", dtype=torch.float32, generator=g)
    expect = main.double().view(N, K) + want if accumulate else want
    if not accumulate:
        main.fill_(float("nan"))
    assert K_.gemm_tn(dy, x, accum_into=main, accumulate=accumulate) is None
    _assert_close(main.view(N, K), expect, f"gemm_tn [{N}x{K}] rows={rows} accumulate={accumulate}")
