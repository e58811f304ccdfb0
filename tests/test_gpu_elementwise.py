"""The memory-bound kernels of the training step (``csrc/elementwise.cu``) against float64 references of the
kernels' own formulas, computed from the same bf16 / fp32 inputs.

Every comparison is per element: ``|got - want| <= atol + rtol * |want|``.  ``rtol`` is the rounding of the output
dtype (``2^-8`` for bf16, ``2^-24`` for fp32); ``atol`` is a first-order bound of the fp32 arithmetic in front of
that rounding, built from the magnitudes of the terms involved.  Bytes the kernels must not write sit in sentinel
margins that must come back bitwise unchanged, and buffers a kernel overwrites start as NaN.

The references are checked against torch's own float64 ops on the CPU, and so are the bounds: the ``*_rejects_*``
tests emulate plausible kernel mistakes in fp32 numpy on the same inputs and require the bound to be exceeded by a
clear margin.  Set ``PIPEGOOSE_ERROR_REPORT=<path>`` to write the largest ``|err| / bound`` of every check to JSON.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

U32 = 2.0 ** -24   # fp32 unit roundoff
UBF = 2.0 ** -8    # bf16 unit roundoff
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    yield
    path = os.environ.get("PIPEGOOSE_ERROR_REPORT")
    if path and _WORST:
        old = {}
        if os.path.exists(path):
            with open(path) as f:
                old = json.load(f)
        old.update(_WORST)
        with open(path, "w") as f:
            json.dump(old, f, indent=1, sort_keys=True)


def _ratio(got, want, atol, rtol):
    """Largest ``|got - want| / (atol + rtol |want|)`` (NaN if ``got`` is NaN where ``want`` is finite)."""
    got, want = got.double(), want.double().to(got.device)
    atol = torch.as_tensor(atol, dtype=torch.float64, device=got.device)
    err = (got - want).abs()
    err = torch.where(got == want, torch.zeros_like(err), err)   # equal infinities
    r = torch.where(err == 0, torch.zeros_like(err), err / (atol + rtol * want.abs()))
    return r.max().item() if r.numel() else 0.0


def _check(name, got, want, atol, rtol):
    r = _ratio(got, want, atol, rtol)
    _WORST[name] = max(_WORST.get(name, 0.0), r)
    assert r <= 1.0, f"{name}: largest |err| / bound is {r:.3g}"


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _f32(x):
    return float(np.float32(x))


def _native():
    from pipegoose_b200 import ops

    return ops.native()


def _split_depth(rows, cols):
    """Longest chain of fp32 additions behind one column of ``colsum`` / LayerNorm ``dgamma``: the launchers split the
    rows over ``rsplit`` blocks of 8 warps (rows strided by 8 per warp), reduce the 8 warps in shared memory and add
    each block's sum with one atomic onto the existing value."""
    cb = (cols + 255) // 256
    rsplit = max(1, min((132 * 4 + cb - 1) // cb, (rows + 63) // 64))
    rpb = (rows + rsplit - 1) // rsplit
    return (rpb + 7) // 8 + 8 + rsplit + 1


# ================================================================================================================
# float64 references
# ================================================================================================================
def ref_layernorm(x, gamma, beta, eps, mean=None, rstd=None):
    """LayerNorm of the rows of ``x``; with ``mean`` / ``rstd`` given, the affine part around those statistics."""
    if mean is None:
        mean = x.mean(-1)
    if rstd is None:
        rstd = 1.0 / torch.sqrt(((x - mean[:, None]) ** 2).mean(-1) + eps)
    return (x - mean[:, None]) * rstd[:, None] * gamma + beta, mean, rstd


def ref_layernorm_bwd(dy, x, gamma, mean, rstd):
    xhat = (x - mean[:, None]) * rstd[:, None]
    g = dy * gamma
    s1 = g.mean(-1, keepdim=True)
    s2 = (g * xhat).mean(-1, keepdim=True)
    return rstd[:, None] * (g - s1 - xhat * s2), (dy * xhat).sum(0), dy.sum(0)


def ref_cross_entropy(logits, targets, ignore_index):
    """Per-row loss and d(loss_row)/d(logits) over the whole vocabulary; ignored rows give 0 and a zero row."""
    ignored = targets == ignore_index
    t = torch.where(ignored, torch.zeros_like(targets), targets)
    lse = torch.logsumexp(logits, -1)
    loss = torch.where(ignored, torch.zeros_like(lse), lse - logits.gather(1, t[:, None]).squeeze(1))
    grad = torch.softmax(logits, -1)
    grad[torch.arange(len(t)), t] -= 1.0
    grad[ignored] = 0.0
    return loss, grad


def ref_adam(p, m, v, g, lr, b1, b2, eps, wd, bc1, bc2, grad_scale, adamw):
    """One Adam (``adamw=False``: L2 decay added to the gradient) or AdamW (decoupled decay) step; returns the new
    ``(p, m, v)`` and the magnitudes the error bounds need."""
    g = g * grad_scale
    G = g.abs()
    if not adamw and wd != 0:
        g = g + wd * p
        G = G + (wd * p).abs()
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    den = torch.sqrt(v / bc2) + eps
    upd = lr * (m / bc1) / den
    if adamw and wd != 0:
        p = p * (1 - lr * wd)
    return p - upd, m, v, dict(G=G, den=den, upd=upd)


def adam_bounds(p0, m0, v0, aux, lr, b1, b2, eps, wd, bc1, bc2, want_m, want_v):
    """Per-element atol of the kernel's fp32 Adam step for master, exp_avg and exp_avg_sq."""
    G, den, upd = aux["G"], aux["den"], aux["upd"]
    at_m = 4 * U32 * (b1 * m0.abs() + (1 - b1) * G)
    at_v = 6 * U32 * (b2 * v0 + (1 - b2) * G * G)
    dv = at_v / bc2
    s = torch.sqrt(want_v / bc2)
    dden = torch.minimum(torch.sqrt(dv), 0.5 * dv / s.clamp_min(1e-300)) + 3 * U32 * den
    at_upd = lr / bc1 * at_m / den + upd.abs() * dden / den + 6 * U32 * upd.abs()
    at_p = 3 * U32 * p0.abs() * (1 + lr * abs(wd)) + at_upd
    return at_p, at_m, at_v


# ================================================================================================================
# CPU: the references against torch's float64 ops
# ================================================================================================================
def test_reference_layernorm_matches_torch():
    g = _gen(0)
    x = torch.randn(37, 264, generator=g, dtype=torch.float64) * 3 + 1
    gamma, beta = torch.randn(264, generator=g, dtype=torch.float64), torch.randn(264, generator=g, dtype=torch.float64)
    dy = torch.randn(37, 264, generator=g, dtype=torch.float64)
    y, mean, rstd = ref_layernorm(x, gamma, beta, 1e-5)
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    yr = torch.nn.functional.layer_norm(xr, (264,), gr, br, 1e-5)
    yr.backward(dy)
    torch.testing.assert_close(y, yr.detach(), rtol=1e-12, atol=1e-12)
    dx, dgamma, dbeta = ref_layernorm_bwd(dy, x, gamma, mean, rstd)
    torch.testing.assert_close(dx, xr.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dgamma, gr.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dbeta, br.grad, rtol=1e-10, atol=1e-10)


def test_reference_cross_entropy_matches_torch():
    g = _gen(1)
    logits = torch.randn(50, 301, generator=g, dtype=torch.float64) * 4
    logits[:, -5:] = -math.inf
    logits[3] *= 300
    targets = torch.randint(0, 296, (50,), generator=g)
    targets[::4] = 0
    loss, grad = ref_cross_entropy(logits, targets, ignore_index=0)
    lr_ = logits.clone().requires_grad_(True)
    want = torch.nn.functional.cross_entropy(lr_, targets, ignore_index=0, reduction="none")
    want.sum().backward()
    torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(grad, lr_.grad, rtol=1e-12, atol=1e-12)
    assert (grad[targets == 0] == 0).all() and (loss[targets == 0] == 0).all()


@pytest.mark.parametrize("adamw", [False, True])
def test_reference_adam_matches_torch(adamw):
    g = _gen(2)
    n, lr, betas, eps, wd, gs = 1000, 1e-2, (0.9, 0.999), 1e-8, 0.1, 0.5
    p0 = torch.randn(n, generator=g, dtype=torch.float64)
    ref = p0.clone().requires_grad_(True)
    opt = (torch.optim.AdamW if adamw else torch.optim.Adam)([ref], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    p, m, v = p0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step in range(1, 6):
        grad = torch.randn(n, generator=g, dtype=torch.float64)
        ref.grad = grad * gs
        opt.step()
        bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
        p, m, v, _ = ref_adam(p, m, v, grad, lr, betas[0], betas[1], eps, wd, bc1, bc2, gs, adamw)
    torch.testing.assert_close(p, ref.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(m, opt.state[ref]["exp_avg"], rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(v, opt.state[ref]["exp_avg_sq"], rtol=1e-12, atol=1e-16)


# ================================================================================================================
# LayerNorm
# ================================================================================================================
def _ln_inputs(rows, h, seed):
    """Rows cycle through: ordinary random, constant (variance 0), large mean (300 +- 1)."""
    g = _gen(seed)
    x = torch.randn(rows, h, generator=g)
    kind = torch.arange(rows) % 3
    x[kind == 1] = torch.randn(int((kind == 1).sum()), 1, generator=g).expand(-1, h)
    x[kind == 2] = 300 + 2 * torch.rand(int((kind == 2).sum()), h, generator=g) - 1
    gamma = 1 + 0.5 * torch.randn(h, generator=g)
    beta = 0.5 * torch.randn(h, generator=g)
    return x.bfloat16(), gamma.bfloat16(), beta.bfloat16()


def _lane_terms(h):
    """Values one lane sums sequentially before the warp's 5-level tree (16-byte chunks strided over 32 lanes)."""
    return 8 * ((h // 8 + 31) // 32)


def _ln_fwd_bounds(x, gamma, beta, eps, mean_k, rstd_k):
    """(want, atol, rtol) for mean, rstd and y.  ``mean`` is checked against the exact mean; ``rstd`` against the
    exact value around the kernel's own mean; ``y`` against the affine part around the kernel's statistics."""
    h = x.shape[1]
    L = _lane_terms(h)
    mean_w = x.mean(-1)
    at_mean = (L + 6) * U32 * x.abs().mean(-1)
    d = x - mean_k[:, None]
    var = (d * d).mean(-1)
    rstd_w = 1.0 / torch.sqrt(var + eps)
    rt_rstd = 0.5 * (L + 12) * U32 + 5 * U32
    y_w, _, _ = ref_layernorm(x, gamma, beta, eps, mean_k, rstd_k)
    at_y = 5 * U32 * (d.abs() * rstd_k[:, None] * gamma.abs() + beta.abs())
    return dict(mean=(mean_w, at_mean, U32), rstd=(rstd_w, 0.0, rt_rstd), y=(y_w, at_y, UBF))


LN_WIDTHS = [8, 264, 2056, 5120, 8192]


@gpu
@pytest.mark.parametrize("rows", [1, 7, 9, 20000])
@pytest.mark.parametrize("h", LN_WIDTHS)
def test_layernorm_fwd_bwd(h, rows):
    from pipegoose_b200.ops import kernels as K

    eps = 1e-5
    xb, gb, bb = (t.cuda() for t in _ln_inputs(rows, h, seed=h + rows))
    y = torch.full((rows, h), math.nan, dtype=torch.bfloat16, device="cuda")
    y, mean, rstd = K.layernorm_fwd(xb, gb, bb, eps, out=y)
    x, gamma, beta = xb.double(), gb.double(), bb.double()
    for name, (want, atol, rtol) in _ln_fwd_bounds(x, gamma, beta, _f32(eps), mean.double(), rstd.double()).items():
        got = {"mean": mean, "rstd": rstd, "y": y}[name]
        _check(f"layernorm_fwd.{name}", got, want, atol, rtol)
    const = torch.arange(rows, device="cuda") % 3 == 1
    assert torch.equal(y[const], bb.expand(rows, h)[const]), "constant rows must come out as beta"

    g = _gen(rows * 7 + h)
    dyb = torch.randn(rows, h, generator=g).bfloat16().cuda()
    extra = torch.randn(rows, h, generator=g).bfloat16().cuda()
    dg0 = torch.randn(h, generator=g).cuda()
    db0 = torch.randn(h, generator=g).cuda()
    dy, mu, rs = dyb.double(), mean.double(), rstd.double()
    dx_w, dg_w, db_w = ref_layernorm_bwd(dy, x, gamma, mu, rs)
    L = _lane_terms(h)
    xhat = (x - mu[:, None]) * rs[:, None]
    dyg = dy * gamma
    s1, s2 = dyg.mean(-1, keepdim=True), (dyg * xhat).mean(-1, keepdim=True)
    ds1 = (L + 7) * U32 * dyg.abs().mean(-1, keepdim=True)
    ds2 = (L + 10) * U32 * (dyg * xhat).abs().mean(-1, keepdim=True)
    at_dx32 = rs[:, None] * (6 * U32 * (dyg.abs() + s1.abs() + (xhat * s2).abs()) + ds1 + xhat.abs() * ds2)
    for with_extra in (False, True):
        dx = torch.full((rows, h), math.nan, dtype=torch.bfloat16, device="cuda")
        dg, db = dg0.clone(), db0.clone()
        K.layernorm_bwd(dyb, xb, gb, mean, rstd, dx_extra=extra if with_extra else None,
                        dgamma_acc=dg, dbeta_acc=db, dx_out=dx)
        want = dx_w + extra.double() if with_extra else dx_w
        at = (1 + UBF) * (at_dx32 + (U32 * extra.double().abs() if with_extra else 0))
        _check("layernorm_bwd.dx", dx, want, at, UBF)
        depth = _split_depth(rows, h)
        _check("layernorm_bwd.dgamma", dg, dg0.double() + dg_w,
               (depth + 4) * U32 * (dg0.double().abs() + (dy * xhat).abs().sum(0)), 0.0)
        _check("layernorm_bwd.dbeta", db, db0.double() + db_w,
               depth * U32 * (db0.double().abs() + dy.abs().sum(0)), 0.0)


def _gather_inputs(seed, V_local=300, h=264, vocab_start=200, rows=600):
    g = _gen(seed)
    table = torch.randn(V_local, h, generator=g).bfloat16()
    gamma = (1 + 0.5 * torch.randn(h, generator=g)).bfloat16()
    beta = (0.5 * torch.randn(h, generator=g)).bfloat16()
    ids = torch.randint(0, vocab_start + V_local + 200, (rows,), generator=g)   # below, inside and above the shard
    ids[:3] = torch.tensor([vocab_start - 1, vocab_start, vocab_start + V_local - 1])
    ids[3] = vocab_start + V_local
    return table, gamma, beta, ids, vocab_start, vocab_start + V_local


@gpu
def test_layernorm_fused_embedding_gather():
    from pipegoose_b200.ops import kernels as K

    table, gamma, beta, ids, vs, ve = (t.cuda() if torch.is_tensor(t) else t for t in _gather_inputs(9))
    y, mean, rstd = K.layernorm_fwd(table, gamma, beta, 1e-5, ids=ids, vocab_start=vs, vocab_end=ve)
    inside = (ids >= vs) & (ids < ve)
    src = torch.where(inside[:, None], table.double()[(ids - vs).clamp(0, table.shape[0] - 1)], 0.0)
    for name, (want, atol, rtol) in _ln_fwd_bounds(src, gamma.double(), beta.double(), _f32(1e-5),
                                                   mean.double(), rstd.double()).items():
        _check(f"layernorm_gather.{name}", {"mean": mean, "rstd": rstd, "y": y}[name], want, atol, rtol)
    assert inside.any() and (~inside).any()
    assert torch.equal(y[~inside], beta.expand(int((~inside).sum()), -1)), "rows outside the shard must be beta"


# ================================================================================================================
# colsum and embedding backward
# ================================================================================================================
@gpu
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 100000])
def test_colsum_strided_accumulates(rows):
    from pipegoose_b200.ops import kernels as K

    cols, ld = 1003, 1024
    g = _gen(rows)
    base = torch.randn(rows, ld, generator=g).bfloat16()
    base[:, cols:] = math.nan   # the last chunk reads past `cols`: those columns must not leak into the sums
    x = base.cuda()[:, :cols]
    out0 = torch.randn(cols, generator=g).cuda()
    buf = torch.full((cols + 16,), -7.0, device="cuda")
    buf[8:8 + cols] = out0
    K.colsum(x, accum_into=buf[8:8 + cols])
    xd = x.double()
    want = out0.double() + xd.sum(0)
    _check("colsum", buf[8:8 + cols], want, _split_depth(rows, cols) * U32 * (out0.double().abs() + xd.abs().sum(0)), 0.0)
    assert (buf[:8] == -7).all() and (buf[8 + cols:] == -7).all()


@gpu
@pytest.mark.parametrize("contended", [False, True])
def test_embedding_bwd(contended):
    from pipegoose_b200.ops import kernels as K

    V_local, h, vs = 300, 264, 200
    rows = 4096 if contended else 700
    g = _gen(11 + contended)
    if contended:
        ids = torch.full((rows,), vs + 7, dtype=torch.int64)   # every row adds into one vocabulary row
    else:
        ids = torch.randint(0, vs + V_local + 200, (rows,), generator=g)
    dx = torch.randn(rows, h, generator=g).bfloat16().cuda()
    ids = ids.cuda()
    dw0 = torch.randn(V_local, h, generator=g).cuda()
    dw = dw0.clone()
    K.embedding_bwd(dx, ids, V_local, vs, vs + V_local, accum_into=dw)
    inside = (ids >= vs) & (ids < vs + V_local)
    loc = (ids - vs)[inside]
    want = dw0.double().index_add(0, loc, dx.double()[inside])
    mag = dw0.double().abs().index_add(0, loc, dx.double().abs()[inside])
    cnt = torch.bincount(loc, minlength=V_local).double()[:, None]
    _check("embedding_bwd.contended" if contended else "embedding_bwd", dw, want, (cnt + 1) * U32 * mag, 0.0)
    assert torch.equal(dw[cnt[:, 0] == 0], dw0[cnt[:, 0] == 0]), "rows no id hit must be unchanged"


# ================================================================================================================
# vocab-parallel cross entropy on virtual ranks
# ================================================================================================================
CE_LAYOUTS = {
    "T1_tail": [1003],                      # one shard, scalar tail of 3
    "T2_tail": [1024, 1001],                # second shard at vocab_start 1024, width not a multiple of 8
    "T3_padshard": [512, 777, 512],         # last shard is all -inf vocabulary padding
}


def _ce_inputs(layout, rows=96, seed=21):
    widths = CE_LAYOUTS[layout]
    V = sum(widths)
    g = _gen(seed)
    logits = torch.randn(rows, V, generator=g) * 3
    logits[1::4] *= 300                      # large magnitudes
    dead = torch.zeros(V, dtype=torch.bool)
    if layout == "T3_padshard":
        dead[V - widths[-1]:] = True
        dead[V - widths[-1] - 6:V - widths[-1] - 2] = True   # inside the last 8-chunk of the middle shard
    else:
        dead[V - 7:V - 2] = True            # in the last full chunk and the tail
    logits[:, dead] = -math.inf
    live = torch.nonzero(~dead).squeeze(1)
    targets = live[torch.randint(0, len(live), (rows,), generator=g)]
    targets[::6] = 0                         # ignore_index 0 is a real token id
    return logits.bfloat16(), targets, widths


def _ce_shards(logits, widths):
    """Each shard in its own 8-padded buffer (NaN padding), handed over as the ``[:, :width]`` view."""
    shards, start = [], 0
    for w in widths:
        buf = torch.full((logits.shape[0], (w + 7) // 8 * 8), math.nan, dtype=torch.bfloat16, device="cuda")
        buf[:, :w] = logits[:, start:start + w]
        shards.append((buf, buf[:, :w], start))
        start += w
    return shards


def _ce_bounds(logits64):
    """Per row, the relative error of the kernels' sum of exponentials: the summation depth plus ``__expf``'s error,
    which grows with |argument| (arguments past -104 underflow in fp32 and contribute nothing)."""
    finite = torch.where(torch.isfinite(logits64), logits64, logits64.new_tensor(math.inf))
    span = (logits64.max(-1).values - finite.min(-1).values).clamp(max=104.0)
    return (64 + 4 * span) * U32


@gpu
@pytest.mark.parametrize("write_grad", [True, False])
@pytest.mark.parametrize("grad_scale", [0.5, None])
@pytest.mark.parametrize("layout", list(CE_LAYOUTS))
def test_cross_entropy_vocab_parallel(layout, grad_scale, write_grad):
    from pipegoose_b200.ops import kernels as K

    logits, targets, widths = _ce_inputs(layout)
    logits, targets = logits.cuda(), targets.cuda()
    shards = _ce_shards(logits, widths)
    before = [buf.clone() for buf, _, _ in shards]
    stats = torch.stack([K.ce_local_stats(view, targets, start) for _, view, start in shards])
    gstats = K.ce_combine_stats(stats) if len(shards) > 1 else stats[0]
    scale_t = None if grad_scale is None else torch.tensor([grad_scale], device="cuda")
    loss = [K.ce_finalize(view, targets, gstats, start, scale_t, ignore_index=0, write_grad=write_grad)
            for _, view, start in shards]
    for l in loss[1:]:
        assert torch.equal(l, loss[0]), "every shard computes the same loss from the global statistics"

    l64 = logits.double()
    want_loss, want_grad = ref_cross_entropy(l64, targets, ignore_index=0)
    eps_s = _ce_bounds(l64)
    gm, tl = l64.max(-1).values, torch.where(targets == 0, 0.0, l64.gather(1, targets[:, None]).squeeze(1))
    at_loss = eps_s + 3 * U32 * (want_loss.abs() + gm.abs() + tl.abs())
    _check("cross_entropy.loss", loss[0], want_loss, at_loss, U32)
    ignored = targets == 0
    assert (loss[0][ignored] == 0).all()
    if not write_grad:
        for (buf, _, _), b in zip(shards, before):
            assert _same_bits(buf, b), "write_grad=False must leave the logits untouched"
        return
    scale = 1.0 if grad_scale is None else grad_scale
    got = torch.cat([view for _, view, _ in shards], dim=1)
    p = torch.softmax(l64, -1)
    at_grad = (1 + UBF) * scale * (2 * eps_s[:, None] * p + 2 * U32)
    _check("cross_entropy.grad", got, want_grad * scale, at_grad, UBF)
    assert (got[ignored] == 0).all(), "ignored rows must get a zero gradient"
    for (buf, view, _), b in zip(shards, before):
        w = view.shape[1]
        assert _same_bits(buf[:, w:], b[:, w:]), "the padding past the shard width must not be written"


@gpu
def test_vocab_parallel_cross_entropy_unaligned_shard_width():
    """A shard width that is not a multiple of 8 (GPT-2's 50257 at TP 2 gives 25129): the loss pads the logits for the
    kernels instead of being refused."""
    from pipegoose_b200.nn.tensor_parallel.loss import VocabParallelCrossEntropy

    class OneRank:
        def get_world_size(self, mode):
            return 1

        def get_local_rank(self, mode):
            return 0

    g = _gen(31)
    B, S, V = 4, 33, 1001
    logits = (torch.randn(B, S, V, generator=g) * 2).bfloat16().cuda().requires_grad_(True)
    tgt = torch.randint(0, V, (B, S), generator=g).cuda()
    loss = VocabParallelCrossEntropy(OneRank())(logits, tgt)
    loss.backward()
    l64 = logits.detach().double().view(-1, V)
    want_loss, want_grad = ref_cross_entropy(l64, tgt.view(-1), ignore_index=-100)
    n = B * S
    eps_s = _ce_bounds(l64)
    assert abs(loss.item() - want_loss.mean().item()) <= (eps_s.max().item() + 8 * U32) * max(1.0, want_loss.mean().item())
    p = torch.softmax(l64, -1)
    _check("cross_entropy.module_v1001.grad", logits.grad.view(-1, V), want_grad / n,
           (1 + UBF) * (2 * eps_s[:, None] * p + 2 * U32) / n, UBF)


@gpu
def test_cross_entropy_refuses_unpadded_rows():
    logits = torch.zeros(4, 1001, dtype=torch.bfloat16, device="cuda")
    stats = torch.empty(4, 3, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 8"):
        _native().ce_stats(logits, torch.zeros(4, dtype=torch.int64, device="cuda"), stats, 0)


# ================================================================================================================
# Adam
# ================================================================================================================
ADAM_HP = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)
ADAM_STEPS = (1, 2, 1000)


def _adam_inputs(n, seed):
    g = _gen(seed)
    p = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * (0.1 if k % 2 else 3.0) for k in range(len(ADAM_STEPS))]
    return p, grads


def _adam_f32_params(step):
    lr, b1, b2, eps = (_f32(ADAM_HP[k]) for k in ("lr", "beta1", "beta2", "eps"))
    bc1, bc2 = _f32(1 - ADAM_HP["beta1"] ** step), _f32(1 - ADAM_HP["beta2"] ** step)
    return lr, b1, b2, eps, bc1, bc2


def _adam_want(p, m, v, g, step, wd, grad_scale, adamw):
    """float64 reference of one kernel step from the kernel's fp32 state, and its bounds."""
    lr, b1, b2, eps, bc1, bc2 = _adam_f32_params(step)
    wd = _f32(wd)
    p, m, v, g = (t.double() for t in (p, m, v, g))
    wp, wm, wv, aux = ref_adam(p, m, v, g, lr, b1, b2, eps, wd, bc1, bc2, _f32(grad_scale), adamw)
    at_p, at_m, at_v = adam_bounds(p, m, v, aux, lr, b1, b2, eps, wd, bc1, bc2, wm, wv)
    return (wp, at_p), (wm, at_m), (wv, at_v)


def _margined(t, margin, fill):
    buf = torch.full((t.numel() + 2 * margin,), fill, dtype=t.dtype, device="cuda")
    buf[margin:margin + t.numel()] = t
    return buf, buf[margin:margin + t.numel()]


@gpu
@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("adamw", [False, True])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1_000_003])
def test_adam_step(n, adamw, wd):
    p0, grads = _adam_inputs(n, seed=n + 10 * adamw + int(100 * wd))
    bufs = {}
    views = {}
    for name, init, fill in (("master", p0, -3.0), ("m", torch.zeros(n), -5.0), ("v", torch.zeros(n), -9.0)):
        bufs[name], views[name] = _margined(init.cuda(), 4, fill)
    pbuf, pview = _margined(p0.bfloat16().cuda(), 4, -2.0)
    for k, step in enumerate(ADAM_STEPS):
        gbuf, gview = _margined(grads[k].cuda(), 4, -11.0)
        state = {name: views[name].clone() for name in views}
        keep = [b.clone() for b in (*bufs.values(), pbuf, gbuf)]
        zero_grad = step == 1
        with_bf16 = step != 2                      # param_bf16 = None must work too
        _native().adam_step(views["master"], views["m"], views["v"], gview, pview if with_bf16 else None,
                            ADAM_HP["lr"], ADAM_HP["beta1"], ADAM_HP["beta2"], ADAM_HP["eps"], wd, step, 0.5, adamw,
                            zero_grad)
        wants = _adam_want(state["master"], state["m"], state["v"], grads[k].cuda(), step, wd, 0.5, adamw)
        for name, (want, atol) in zip(("master", "m", "v"), wants):
            _check(f"adam.{name}", views[name], want, atol, U32)
        if with_bf16:
            assert _same_bits(pview, views["master"].bfloat16()), "param_bf16 must be master rounded to bf16"
        assert torch.equal(gview, torch.zeros_like(gview)) if zero_grad else _same_bits(gview, grads[k].cuda())
        for b, kb in zip((*bufs.values(), pbuf, gbuf), keep):
            assert _same_bits(b[:4], kb[:4]) and _same_bits(b[-4:], kb[-4:]), "write outside the n elements"


@gpu
@pytest.mark.parametrize("zero_grad", [False, True])
@pytest.mark.parametrize("stride_kind", ["packed", "world"])
@pytest.mark.parametrize("seg", [4, 128, 1000])
@pytest.mark.parametrize("nb", [1, 3, 7])
def test_adam_step_strided_matches_per_slice(nb, seg, stride_kind, zero_grad):
    world, rank = 3, 1
    stride = seg if stride_kind == "packed" else world * seg
    first = rank * seg
    total = first + (nb - 1) * stride + seg + 2 * seg + 8
    g = _gen(nb * 1000 + seg)
    flat_grad = torch.randn(total, generator=g).cuda()
    flat_param = torch.randn(total, generator=g).bfloat16().cuda()
    master = torch.randn(nb * seg, generator=g).cuda()
    m = (0.1 * torch.randn(nb * seg, generator=g)).cuda()
    v = torch.rand(nb * seg, generator=g).cuda() * 0.01
    hp = (ADAM_HP["lr"], ADAM_HP["beta1"], ADAM_HP["beta2"], ADAM_HP["eps"], 0.1, 7, 0.5, True, zero_grad)

    ref = [t.clone() for t in (master, m, v, flat_grad, flat_param)]
    for b in range(nb):
        s = first + b * stride
        _native().adam_step(ref[0][b * seg:(b + 1) * seg], ref[1][b * seg:(b + 1) * seg], ref[2][b * seg:(b + 1) * seg],
                            ref[3][s:s + seg], ref[4][s:s + seg], *hp)
    got = [t.clone() for t in (master, m, v, flat_grad, flat_param)]
    _native().adam_step_strided(got[0], got[1], got[2], got[3], got[4], first, seg, stride, nb, *hp)
    for a, b in zip(got, ref):
        assert _same_bits(a, b), "the strided launch must equal one adam_step per slice, bitwise"
    owned = torch.zeros(total, dtype=torch.bool, device="cuda")
    for b in range(nb):
        owned[first + b * stride:first + b * stride + seg] = True
    assert _same_bits(got[3][~owned], flat_grad[~owned]) and _same_bits(got[4][~owned], flat_param[~owned])
    assert not _same_bits(got[4][owned], flat_param[owned])


@gpu
@pytest.mark.parametrize("groups", [1, 2])
def test_fused_adam_zero1_shard(groups):
    """FusedAdam owning slice 1 of 2 of every bucket (ZeRO-1), on one GPU: with one parameter group the equal bucket
    slices go through one strided launch, with two (decay / no decay) through the per-group plan."""
    from pipegoose_b200.optim import FusedAdam

    g = _gen(40 + groups)
    shapes = [(96, 40), (40,), (40,), (200, 40), (40,), (33, 7)]
    params = [torch.nn.Parameter(torch.randn(s, generator=g).bfloat16().cuda()) for s in shapes]
    decay = [p for p in params if p.dim() >= 2]
    no_decay = [p for p in params if p.dim() < 2]
    lr, wd = 1e-2, 0.1
    if groups == 1:
        opt = FusedAdam(params, lr=lr, weight_decay=wd, adamw=True)
    else:
        opt = FusedAdam([{"params": decay}, {"params": no_decay, "weight_decay": 0.0}], lr=lr, weight_decay=wd, adamw=True)
    flat = opt.ensure_flat()
    opt.set_bucket_shards(1024, rank=1, world=2)
    owned = torch.zeros(flat.numel, dtype=torch.bool)
    for s, e in opt._segments:
        owned[s:e] = True
    wd_of = torch.zeros(flat.numel, dtype=torch.float64)
    in_param = torch.zeros(flat.numel, dtype=torch.bool)
    for p in params:
        o, n = flat.param_range(p)
        in_param[o:o + n] = True
        wd_of[o:o + n] = wd if (groups == 1 or p.dim() >= 2) else 0.0
    p64 = flat.flat_param.double().cpu()
    m64, v64 = torch.zeros_like(p64), torch.zeros_like(p64)
    start = flat.flat_param.clone()
    b1, b2 = 0.9, 0.999
    for step in (1, 2):
        grad = torch.randn(flat.numel, generator=g) * in_param
        flat.flat_grad.copy_(grad)
        opt.step()
        g64 = grad.double()
        m64 = b1 * m64 + (1 - b1) * g64
        v64 = b2 * v64 + (1 - b2) * g64 * g64
        p64 = p64 * (1 - lr * wd_of) - lr * (m64 / (1 - b1 ** step)) / (torch.sqrt(v64 / (1 - b2 ** step)) + 1e-8)
    master = torch.cat([p64[s:e] for s, e in opt._segments])
    # two steps of fp32 arithmetic: each update is at most a few lr, computed to a few tens of ulp
    _check(f"fused_adam.groups{groups}", opt.master, master, 256 * U32 * lr + 4 * U32 * master.abs(), 0.0)
    got = flat.flat_param.cpu()
    assert _same_bits(got[~owned], start.cpu()[~owned]), "parameters outside the owned slices must be untouched"
    assert _same_bits(got[owned], opt.master.cpu().bfloat16()), "owned parameters are the bf16 master"


@gpu
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("n", list(range(1, 18)) + [8191, 8192, 8193])
def test_accum_bf16_to_f32(n, accumulate):
    g = _gen(n + 100 * accumulate)
    src = torch.randn(n, generator=g).bfloat16().cuda()
    d0 = torch.randn(n, generator=g).cuda()
    sbuf, sview = _margined(src, 8, -1.0)
    dbuf, dview = _margined(d0 if accumulate else torch.full((n,), math.nan, device="cuda"), 4, -13.0)
    keep = dbuf.clone()
    scale = 0.3
    _native().accum_bf16_to_f32(sview, dview, scale, accumulate)
    t = src.double() * _f32(scale)
    want = d0.double() + t if accumulate else t
    _check("accum_bf16_to_f32", dview, want, 2 * U32 * (t.abs() + (d0.double().abs() if accumulate else 0)), 0.0)
    assert _same_bits(dbuf[:4], keep[:4]) and _same_bits(dbuf[-4:], keep[-4:])


# ================================================================================================================
# preconditions the bindings refuse (each check runs before any launch)
# ================================================================================================================
@gpu
@pytest.mark.parametrize("which", ["master", "m", "v", "grad", "param_bf16"])
def test_adam_step_refuses_misaligned(which):
    n = 64
    t = {k: torch.zeros(n + 4, device="cuda") for k in ("master", "m", "v", "grad")}
    pb = torch.zeros(n + 4, dtype=torch.bfloat16, device="cuda")
    args = {k: t[k][:n] for k in t}
    args["param_bf16"] = pb[:n]
    args[which] = (pb if which == "param_bf16" else t[which])[1:n + 1]
    with pytest.raises(RuntimeError, match="aligned"):
        _native().adam_step(args["master"], args["m"], args["v"], args["grad"], args["param_bf16"],
                            1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, False)


@gpu
@pytest.mark.parametrize("which", ["first", "master", "flat_grad", "flat_param"])
def test_adam_step_strided_refuses_misaligned(which):
    seg, nb = 8, 2
    master, m, v = (torch.zeros(seg * nb + 4, device="cuda") for _ in range(3))
    grad = torch.zeros(64, device="cuda")
    param = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    first = 2 if which == "first" else 0
    args = [master[:seg * nb], m[:seg * nb], v[:seg * nb], grad[:60], param[:60]]
    if which == "master":
        args[0] = master[1:seg * nb + 1]
    elif which == "flat_grad":
        args[3] = grad[1:61]
    elif which == "flat_param":
        args[4] = param[1:61]
        args[3] = grad[:60]
    with pytest.raises(RuntimeError, match="aligned|multiple of 4"):
        _native().adam_step_strided(*args, first, seg, 16, nb, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, False, False)


@gpu
@pytest.mark.parametrize("which", ["src", "dst"])
def test_accum_bf16_to_f32_refuses_misaligned(which):
    src = torch.zeros(40, dtype=torch.bfloat16, device="cuda")
    dst = torch.zeros(40, device="cuda")
    s, d = (src[1:33], dst[:32]) if which == "src" else (src[:32], dst[1:33])
    with pytest.raises(RuntimeError, match="aligned"):
        _native().accum_bf16_to_f32(s, d, 1.0, True)


@gpu
def test_embedding_bwd_refuses_width_not_multiple_of_8():
    dx = torch.zeros(4, 12, dtype=torch.bfloat16, device="cuda")
    dw = torch.zeros(10, 12, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 8"):
        _native().embedding_bwd(dx, torch.zeros(4, dtype=torch.int64, device="cuda"), dw, 0, 10)


# ================================================================================================================
# CPU: the bounds reject plausible kernel mistakes (fp32 numpy emulations on the GPU tests' own inputs)
# ================================================================================================================
MARGIN = 4.0   # a mistake must exceed its bound at least this many times over


def _np_adam(p, m, v, g, step, wd, gs, adamw, swap_bc=False, swap_decay=False, scale_late=False):
    """The kernel's fp32 Adam step in numpy, optionally with one mistake."""
    lr, b1, b2, eps, bc1, bc2 = (np.float32(x) for x in _adam_f32_params(step))
    if swap_bc:
        bc1, bc2 = bc2, bc1
    wd, gs = np.float32(wd), np.float32(gs)
    if swap_decay:
        adamw = not adamw
    g = g if scale_late else g * gs
    if not adamw and wd != 0:
        g = g + wd * p
    m = b1 * m + (np.float32(1) - b1) * g
    v = b2 * v + (np.float32(1) - b2) * g * g
    upd = lr * (m / bc1) / (np.sqrt(v / bc2) + eps)
    if scale_late:
        upd = upd * gs
    if adamw and wd != 0:
        p = p * (np.float32(1) - lr * wd)
    return p - upd, m, v


@pytest.mark.parametrize("mistake", ["swap_bc", "swap_decay", "scale_late"])
def test_adam_bounds_reject_mistakes(mistake):
    n, wd, gs = 1_000_003, 0.1, 0.5
    worst = math.inf
    for adamw in (False, True):
        p0, grads = _adam_inputs(n, seed=n + 10 * adamw + int(100 * wd))
        p, m, v = p0.numpy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
        for k, step in enumerate(ADAM_STEPS):
            gk = grads[k].numpy()
            wants = _adam_want(torch.from_numpy(p), torch.from_numpy(m), torch.from_numpy(v), grads[k], step, wd, gs, adamw)
            bad = _np_adam(p, m, v, gk, step, wd, gs, adamw, **{mistake: True})
            r = max(_ratio(torch.from_numpy(b), w, a, U32) for b, (w, a) in zip(bad, wants))
            worst = min(worst, r)
            p, m, v = _np_adam(p, m, v, gk, step, wd, gs, adamw)
            good = max(_ratio(torch.from_numpy(b), w, a, U32) for b, (w, a) in zip((p, m, v), wants))
            assert good <= 1.0, "the correct emulation must pass its own bound"
    print(f"adam {mistake}: smallest over cases of the largest |err| / bound = {worst:.3g}")
    assert worst > MARGIN


def test_adam_bound_rejects_a_dropped_tail_element():
    n = 5
    p0, grads = _adam_inputs(n, seed=n + 10 + 10)
    p, m, v = p0.numpy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    (want, at), _, _ = _adam_want(p0, torch.zeros(n), torch.zeros(n), grads[0], 1, 0.1, 0.5, True)
    bad = _np_adam(p, m, v, grads[0].numpy(), 1, 0.1, 0.5, True)[0]
    bad[-1] = p[-1]                              # the scalar tail left un-updated
    r = _ratio(torch.from_numpy(bad), want, at, U32)
    print(f"adam dropped tail element: largest |err| / bound = {r:.3g}")
    assert r > MARGIN


def test_layernorm_bound_rejects_biased_variance():
    """``1/(h-1)`` instead of ``1/h`` in the variance, at the widest row (where the change is smallest)."""
    worst = math.inf
    for h in LN_WIDTHS:
        xb, gb, bb = _ln_inputs(9, h, seed=h + 9)
        x = xb.numpy().astype(np.float32) if xb.dtype != torch.bfloat16 else xb.float().numpy()
        mean = x.mean(-1, dtype=np.float32)
        var = ((x - mean[:, None]) ** 2).sum(-1, dtype=np.float32) / np.float32(h - 1)
        rstd = (np.float32(1) / np.sqrt(var + np.float32(1e-5))).astype(np.float32)
        b = _ln_fwd_bounds(xb.double(), gb.double(), bb.double(), _f32(1e-5), torch.from_numpy(mean).double(),
                           torch.from_numpy(rstd).double())
        want, atol, rtol = b["rstd"]
        worst = min(worst, _ratio(torch.from_numpy(rstd), want, atol, rtol))
    print(f"layernorm 1/(h-1): smallest over widths of the largest |err| / bound = {worst:.3g}")
    assert worst > MARGIN


def test_gather_bound_rejects_ignored_vocab_start():
    table, gamma, beta, ids, vs, ve = _gather_inputs(9)
    t = table.float().numpy()
    ok = (ids >= vs) & (ids < ve)
    bad_src = np.where(ok.numpy()[:, None], t[np.clip(ids.numpy(), 0, len(t) - 1)], 0).astype(np.float32)  # id, not id - vs
    mean = bad_src.mean(-1, dtype=np.float32)
    rstd = (1 / np.sqrt(((bad_src - mean[:, None]) ** 2).mean(-1) + np.float32(1e-5))).astype(np.float32)
    src = torch.where(ok[:, None], table.double()[(ids - vs).clamp(0, table.shape[0] - 1)], 0.0)
    b = _ln_fwd_bounds(src, gamma.double(), beta.double(), _f32(1e-5), torch.from_numpy(mean).double(),
                       torch.from_numpy(rstd).double())
    r = _ratio(torch.from_numpy(mean), *b["mean"])
    print(f"layernorm gather, vocab_start ignored: largest |err| / bound of the mean = {r:.3g}")
    assert r > MARGIN


def _np_ce_loss(l, targets, widths, vocab_start_ignored=False, drop_tail=False):
    """The kernels' per-row loss in fp32 numpy: per-shard (max, sumexp, target logit), merged across shards."""
    ms, ss, ts, start = [], [], [], 0
    for w in widths:
        sh = l[:, start:start + w].copy()
        if drop_tail and w % 8:
            sh = sh[:, :w - 1]
        with np.errstate(invalid="ignore", over="ignore"):
            m = sh.max(-1)
            s = np.where(np.isfinite(m), np.exp(sh - np.where(np.isfinite(m), m, 0)[:, None]).sum(-1), 0).astype(np.float32)
        t = targets - (0 if vocab_start_ignored else start)
        ok = (t >= 0) & (t < w)
        ts.append(np.where(ok, sh[np.arange(len(t)), np.clip(t, 0, sh.shape[1] - 1)], 0).astype(np.float32))
        ms.append(m)
        ss.append(s)
        start += w
    M = np.max(ms, 0)
    S = sum(np.where(np.isfinite(mi), si * np.exp(mi - M), 0) for mi, si in zip(ms, ss)).astype(np.float32)
    return np.where(targets == 0, 0, np.log(S) + M - sum(ts)).astype(np.float32)


@pytest.mark.parametrize("mistake", ["vocab_start_ignored", "drop_tail"])
def test_cross_entropy_bound_rejects_mistakes(mistake):
    layout = "T2_tail"
    logits, targets, widths = _ce_inputs(layout)
    l = logits.float().numpy()
    bad = _np_ce_loss(l, targets.numpy(), widths, **{mistake: True})
    good = _np_ce_loss(l, targets.numpy(), widths)
    l64 = logits.double()
    want, _ = ref_cross_entropy(l64, targets, ignore_index=0)
    eps_s = _ce_bounds(l64)
    gm, tl = l64.max(-1).values, torch.where(targets == 0, 0.0, l64.gather(1, targets[:, None]).squeeze(1))
    at = eps_s + 3 * U32 * (want.abs() + gm.abs() + tl.abs())
    assert _ratio(torch.from_numpy(good), want, at, U32) <= 1.0, "the correct emulation must pass its own bound"
    r = _ratio(torch.from_numpy(bad), want, at, U32)
    print(f"cross entropy {mistake}: largest |err| / bound of the loss = {r:.3g}")
    assert r > MARGIN
