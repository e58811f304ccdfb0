"""The fused MoE path on one GPU: router, dispatch, grouped expert GEMMs, scatter-combine and ``FusedExpertLayer``.

Dispatch and the scatter-combine address their destinations through plain device pointers (NVLink peer mappings in
a real expert-parallel group), so T ordinary local buffer sets stand in for T ranks here ("virtual ranks").  The whole
layer runs in a one-process NCCL group, where the symmetric workspace has no peers to open.
"""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_GELU, EPI_DGELU, EPI_SCATTER = 2, 32, 64


def _C():
    from pipegoose_b200 import ops

    return ops.native()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ moe_route
def _route(x, wg, bg, jitter, top_k, capacity):
    n, E = x.shape[0], wg.shape[0]
    dev = x.device
    out = dict(probs=torch.empty(n, E, dtype=torch.float32, device=dev),
               topk_idx=torch.empty(n, top_k, dtype=torch.int32, device=dev),
               topk_prob=torch.empty(n, top_k, dtype=torch.float32, device=dev),
               pos=torch.empty(n, top_k, dtype=torch.int32, device=dev),
               counts=torch.zeros(E, dtype=torch.int32, device=dev),
               prob_sum=torch.zeros(E, dtype=torch.float32, device=dev),
               zsum=torch.zeros(1, dtype=torch.float32, device=dev),
               lse=torch.empty(n, dtype=torch.float32, device=dev))
    _C().moe_route(x, wg, bg, jitter, top_k, capacity, out["probs"], out["topk_idx"], out["topk_prob"], out["pos"],
                   out["counts"], out["prob_sum"], out["zsum"], out["lse"])
    return out


def _route_inputs(n, h, E, bias, jitter, seed):
    g = _gen(seed)
    x = torch.randn(n, h, device="cuda", dtype=torch.bfloat16, generator=g)
    wg = (torch.randn(E, h, device="cuda", generator=g) * (2.0 / h ** 0.5)).to(torch.bfloat16)
    bg = (torch.randn(E, device="cuda", generator=g) * 0.5).to(torch.bfloat16) if bias else None
    jt = (torch.rand(n, E, device="cuda", generator=g) * 0.2 + 0.9) if jitter else None
    return x, wg, bg, jt


def _route_reference(x, wg, bg, jitter):
    logits = x.double() @ wg.double().t()
    if bg is not None:
        logits = logits + bg.double()
    if jitter is not None:
        logits = logits * jitter.double()
    return torch.softmax(logits, -1), torch.logsumexp(logits, -1)


def _check_slots(r, E, capacity):
    """counts = histogram of the chosen experts (dropped ones included); per expert the kept slots are exactly
    0 .. min(count, C) - 1 and the rest are -1."""
    idx, pos = r["topk_idx"].long().flatten(), r["pos"].flatten()
    hist = torch.bincount(idx, minlength=E)
    assert torch.equal(r["counts"].long(), hist), (r["counts"], hist)
    for e in range(E):
        p = pos[idx == e]
        cnt = int(hist[e])
        kept = torch.sort(p[p >= 0]).values
        assert torch.equal(kept, torch.arange(min(cnt, capacity), device=p.device, dtype=p.dtype)), e
        assert int((p == -1).sum()) == max(0, cnt - capacity), e


@pytest.mark.parametrize("n", [1, 7, 1000, 8192])
@pytest.mark.parametrize("h", [64, 1024, 2560])
@pytest.mark.parametrize("E", [2, 4, 6, 16, 20, 64])
def test_moe_route(E, h, n):
    """Gate GEMV, softmax, top-k, capacity slots and the loss partial sums against float64, with and without a gate
    bias and jitter, top-1 and top-2; the jittered runs use a capacity small enough to drop tokens."""
    if E * h * 2 > 200 * 1024:
        x, wg, _, _ = _route_inputs(8, h, E, False, False, seed=1)
        with pytest.raises(RuntimeError):  # the gate matrix does not fit in shared memory: refused before launch
            _route(x, wg, None, None, 1, 8)
        return
    for (bias, jitter), top_k in itertools.product([(False, False), (True, False), (False, True), (True, True)], [1, 2]):
        x, wg, bg, jt = _route_inputs(n, h, E, bias, jitter, seed=E * 1000 + h + n + 7 * bias + 3 * jitter)
        capacity = n * top_k if not jitter else max(1, (n * top_k) // (2 * E))
        r = _route(x, wg, bg, jt, top_k, capacity)
        p_ref, lse_ref = _route_reference(x, wg, bg, jt)
        what = f"E={E} h={h} n={n} top_k={top_k} bias={bias} jitter={jitter}"
        assert (r["probs"].double() - p_ref).abs().max().item() <= 1e-5, what
        assert (r["lse"].double() - lse_ref).abs().max().item() <= 1e-5 * max(1.0, lse_ref.abs().max().item()), what
        assert torch.allclose(r["prob_sum"].double(), p_ref.sum(0), rtol=1e-4, atol=1e-4), what
        assert torch.allclose(r["zsum"].double(), lse_ref.square().sum(), rtol=1e-4), what
        # top-k against torch.topk, except where the k-th and (k+1)-th probabilities are too close to call
        top = torch.topk(p_ref, min(top_k + 1, E), dim=-1)
        gaps = top.values[:, :-1] - top.values[:, 1:]
        clear = (gaps[:, :top_k] > 1e-4).all(-1) if top_k < E else (gaps > 1e-4).all(-1)
        assert torch.equal(r["topk_idx"].long()[clear], top.indices[clear, :top_k]), what
        assert torch.equal(r["topk_prob"], r["probs"].gather(1, r["topk_idx"].long())), what
        _check_slots(r, E, capacity)


@pytest.mark.parametrize("top_k", [1, 2])
def test_moe_route_matches_eager_router(top_k):
    """Same probabilities, Switch aux loss and z-loss as the eager ``_TopKRouter`` (``Top1Router`` / ``Top2Router``)."""
    from pipegoose_b200.nn.expert_parallel import Top1Router, Top2Router

    n, h, E, alpha = 1000, 1024, 6, 0.01
    x, wg, bg, _ = _route_inputs(n, h, E, True, False, seed=40 + top_k)
    router = (Top1Router if top_k == 1 else Top2Router)(None, E, h, alpha=alpha).cuda().eval()
    with torch.no_grad():
        router.gate.weight.copy_(wg.float())
        router.gate.bias.copy_(bg.float())
        eager = router(x)
    r = _route(x, wg, bg, None, top_k, n * top_k)
    mask = torch.zeros(n, E, device="cuda").scatter_(1, r["topk_idx"].long(), 1.0)
    assert torch.equal(mask, eager.dispatching_order)
    assert torch.allclose(r["probs"] * mask, eager.weight, rtol=1e-5, atol=1e-6)
    aux = alpha * E * torch.dot(r["counts"].float() / n, r["prob_sum"] / n)
    assert torch.allclose(aux, eager.aux_loss, rtol=1e-4), (aux, eager.aux_loss)
    assert torch.allclose(r["zsum"][0] / n, eager.z_loss, rtol=1e-4), (r["zsum"][0] / n, eager.z_loss)


def test_moe_route_non_finite_tokens():
    """A token whose gate input is NaN or +-inf is dropped for every k (expert 0, weight 0, no slot, not counted);
    its NaN still reaches probs, lse and the loss partial sums.  The other tokens are routed as usual."""
    n, h, E, top_k = 64, 256, 4, 2
    x, wg, bg, _ = _route_inputs(n, h, E, True, False, seed=50)
    bad = [3, 17, 40]
    x[3, 5] = float("nan")
    x[17, 100] = float("inf")
    x[40, 0] = float("-inf")
    r = _route(x, wg, bg, None, top_k, n * top_k)
    good = torch.ones(n, dtype=torch.bool, device="cuda")
    good[bad] = False
    assert torch.isnan(r["probs"][bad]).all() and torch.isnan(r["lse"][bad]).all()
    assert torch.isnan(r["zsum"]).all() and torch.isnan(r["prob_sum"]).all()
    assert bool((r["pos"][bad] == -1).all()) and bool((r["topk_idx"][bad] == 0).all())
    assert bool((r["topk_prob"][bad] == 0).all())
    assert torch.equal(r["counts"].long(), torch.bincount(r["topk_idx"][good].long().flatten(), minlength=E))
    p_ref, _ = _route_reference(x[good], wg, bg, None)
    assert (r["probs"][good].double() - p_ref).abs().max().item() <= 1e-5
    assert bool((r["pos"][good] >= 0).all())


@pytest.mark.parametrize("E,top_k", [(1, 2), (4, 3), (2, 0)])
def test_moe_route_rejects_bad_top_k(E, top_k):
    x, wg, _, _ = _route_inputs(16, 64, E, False, False, seed=60)
    with pytest.raises(RuntimeError):
        _route(x, wg, None, None, top_k, 32)


# ------------------------------------------------------------------------------------------------ moe_dispatch
def _virtual_ranks(T, rows, h, El):
    return [dict(buf=torch.zeros(rows, h, device="cuda", dtype=torch.bfloat16),
                 ret=torch.full((rows,), -1, device="cuda", dtype=torch.int32),
                 scale=torch.ones(rows, device="cuda", dtype=torch.float32),
                 arrive=torch.zeros(El, device="cuda", dtype=torch.int32)) for _ in range(T)]


def _dispatch(x, r, ranks, top_k, El, C, my_rank, scale_by_prob, blocks):
    _C().moe_dispatch(x, r["topk_idx"], r["topk_prob"], r["pos"], [v["buf"].data_ptr() for v in ranks],
                      [v["ret"].data_ptr() for v in ranks], [v["scale"].data_ptr() for v in ranks],
                      [v["arrive"].data_ptr() for v in ranks], top_k, El, C, my_rank, scale_by_prob, blocks)


@pytest.mark.parametrize("scale_by_prob", [False, True])
@pytest.mark.parametrize("T,my_rank", [(1, 0), (2, 0), (2, 1), (4, 0), (4, 3)])
def test_moe_dispatch_virtual_ranks(T, my_rank, scale_by_prob):
    """Every kept (token, k) lands in buf[owner][e_local * T*C + my_rank * C + pos], bitwise, with its return address
    k*n + t and gate weight; nothing else is written; every arrival counter reaches ``blocks``."""
    n, h, El, top_k, blocks = 700, 256, 2, 2, 16
    E = El * T
    C = max(1, (n * top_k) // (2 * E))  # drops some tokens
    x, wg, bg, _ = _route_inputs(n, h, E, True, False, seed=70 + T)
    r = _route(x, wg, bg, None, top_k, C)
    rows = El * T * C
    ranks = _virtual_ranks(T, rows, h, El)
    _dispatch(x, r, ranks, top_k, El, C, my_rank, scale_by_prob, blocks)

    want_buf = torch.zeros(T * rows, h, device="cuda", dtype=torch.bfloat16)
    want_ret = torch.full((T * rows,), -1, device="cuda", dtype=torch.int32)
    want_scale = torch.ones(T * rows, device="cuda", dtype=torch.float32)
    idx, pos, prob = r["topk_idx"].long(), r["pos"].long(), r["topk_prob"]
    t_ix, k_ix = torch.nonzero(pos >= 0, as_tuple=True)
    e = idx[t_ix, k_ix]
    owner, el = e // El, e % El
    grow = owner * rows + el * (T * C) + my_rank * C + pos[t_ix, k_ix]
    p = prob[t_ix, k_ix]
    want_buf[grow] = (x[t_ix].float() * p[:, None]).to(torch.bfloat16) if scale_by_prob else x[t_ix]
    want_ret[grow] = (k_ix * n + t_ix).int()
    want_scale[grow] = p
    assert t_ix.numel() < n * top_k  # some were dropped
    assert torch.equal(torch.cat([v["buf"] for v in ranks]), want_buf)
    assert torch.equal(torch.cat([v["ret"] for v in ranks]), want_ret)
    assert torch.equal(torch.cat([v["scale"] for v in ranks]), want_scale)
    for v in ranks:
        assert bool((v["arrive"] == blocks).all()), v["arrive"]


@pytest.mark.parametrize("T", [0, 9])
def test_moe_dispatch_rejects_bad_peer_lists(T):
    n, h, top_k = 16, 64, 1
    x, wg, _, _ = _route_inputs(n, h, 2, False, False, seed=80)
    r = _route(x, wg, None, None, top_k, n)
    ranks = _virtual_ranks(max(T, 1), 128, h, 1)[:T] if T else []
    with pytest.raises(RuntimeError, match="peer"):
        _dispatch(x, r, ranks, top_k, 1, 64, 0, False, 4)
    two = _virtual_ranks(2, 128, h, 1)
    with pytest.raises(RuntimeError, match="same length"):
        _C().moe_dispatch(x, r["topk_idx"], r["topk_prob"], r["pos"], [v["buf"].data_ptr() for v in two],
                          [two[0]["ret"].data_ptr()], [v["scale"].data_ptr() for v in two],
                          [v["arrive"].data_ptr() for v in two], top_k, 1, 64, 0, False, 4)


# ------------------------------------------------------------------------------------------------ grouped GEMMs
def _expert_weights(El, h, f, seed):
    g = _gen(seed)
    w1 = (torch.randn(El, f, h, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b1 = (torch.randn(El, f, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w2 = (torch.randn(El, h, f, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b2 = (torch.randn(El, h, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return w1, b1, w2, b2


@pytest.mark.parametrize("block_n", [0, 128, 256])
def test_grouped_fc1_gelu_bias_bit_identical(block_n):
    """Grouped fc1 (one chunk per expert, stacked weights, per-chunk bias, GELU + pre-activation) is bitwise equal to
    per-expert plain GEMMs: the main loop is shared, and both epilogues give the same bits."""
    from pipegoose_b200.ops import kernels as K_

    El, R, h, f = 4, 256, 256, 1024
    w1, b1, _, _ = _expert_weights(El, h, f, seed=90)
    xbuf = torch.randn(El * R, h, device="cuda", generator=_gen(91)).to(torch.bfloat16)
    h1 = torch.empty(El * R, f, device="cuda", dtype=torch.bfloat16)
    z = torch.empty(El * R, f, device="cuda", dtype=torch.bfloat16)
    _C().gemm(xbuf, w1.view(El * f, h), h1, False, False, b1.view(-1), None, z, EPI_GELU, block_n, 0, El, 0, 0, 0,
              [], [], dict(b_chunk_rows=f, bias_chunk_stride=f))
    for e in range(El):
        sl = slice(e * R, (e + 1) * R)
        z_e = torch.empty(R, f, device="cuda", dtype=torch.bfloat16)
        h_e = K_.gemm_nt(xbuf[sl], w1[e], b1[e], gelu=True, aux_out=z_e, block_n=block_n)
        assert torch.equal(h1[sl], h_e), e
        assert torch.equal(z[sl], z_e), e


@pytest.mark.parametrize("block_n", [0, 128, 256])
def test_grouped_fc2_dgrad_dgelu_bit_identical(block_n):
    """Grouped backward through fc2 (B MN-major, GELU' epilogue) is bitwise equal to per-expert ``gemm_nn``."""
    from pipegoose_b200.ops import kernels as K_

    El, R, h, f = 4, 256, 256, 1024
    _, _, w2, _ = _expert_weights(El, h, f, seed=92)
    dybuf = torch.randn(El * R, h, device="cuda", generator=_gen(93)).to(torch.bfloat16)
    z = torch.randn(El * R, f, device="cuda", generator=_gen(94)).to(torch.bfloat16)
    dz = torch.empty(El * R, f, device="cuda", dtype=torch.bfloat16)
    _C().gemm(dybuf, w2.view(El * h, f), dz, False, True, None, None, z, EPI_DGELU, block_n, 0, El, 0, 0, 0, [], [],
              dict(b_chunk_rows=h))
    for e in range(El):
        sl = slice(e * R, (e + 1) * R)
        assert torch.equal(dz[sl], K_.gemm_nn(dybuf[sl], w2[e], dgelu_aux=z[sl], block_n=block_n)), e


@pytest.mark.parametrize("block_n", [64, 128, 256])
@pytest.mark.parametrize("T", [1, 2, 4])
def test_scatter_combine_virtual_sources(T, block_n):
    """EPI_SCATTER: row r of expert chunk e goes to comb[(r - e*T*C) // C][row_ret[r]] as bf16((fp32 GEMM + bias) *
    row_scale[r]).  The fp32 GEMM comes from the fp32-output form of the same call (same main loop and tile width),
    and the epilogue's fp32 bias add and scale are repeated in the same order, so the rows match bitwise.  Rows whose
    row_ret is -1 go nowhere; every row of every buffer that no row_ret points at stays bitwise untouched."""
    El, C, h, f, top_k, n = 3, 128, 256, 512, 2, 400
    R = T * C
    _, _, w2, b2 = _expert_weights(El, h, f, seed=100 + T)
    g = _gen(101 + T)
    h1 = torch.randn(El * R, f, device="cuda", generator=g).to(torch.bfloat16)
    scale = torch.rand(El * R, device="cuda", generator=g) + 0.25
    ret = torch.full((El * R,), -1, device="cuda", dtype=torch.int32)
    for s in range(T):
        rows_s = torch.cat([torch.arange(e * R + s * C, e * R + (s + 1) * C, device="cuda") for e in range(El)])
        addr = torch.randperm(top_k * n, device="cuda", generator=g)[:rows_s.numel()].int()
        keep = torch.rand(rows_s.numel(), device="cuda", generator=g) > 0.25   # holes
        ret[rows_s[keep]] = addr[keep]
    sentinel = torch.randn(top_k * n, h, device="cuda", generator=g).to(torch.bfloat16)
    comb = [sentinel.clone() for _ in range(T)]
    dummy = torch.empty(1, h, device="cuda", dtype=torch.bfloat16)
    _C().gemm(h1, w2.view(El * h, f), dummy, False, False, b2.view(-1), None, None, EPI_SCATTER, block_n, 0, El, 0, 0, 0,
              [c.data_ptr() for c in comb], [],
              dict(b_chunk_rows=h, bias_chunk_stride=h, row_ret=ret.data_ptr(), row_scale=scale.data_ptr(),
                   rows_per_src=C))
    want = [sentinel.clone() for _ in range(T)]
    for e in range(El):
        sl = slice(e * R, (e + 1) * R)
        acc = torch.empty(R, h, device="cuda", dtype=torch.float32)
        _C().gemm(h1[sl], w2[e], acc, False, False, None, None, None, 0, block_n, 0, ag={"k_splits": 1})
        rows = ((acc + b2[e].float()) * scale[sl, None]).to(torch.bfloat16)
        for s in range(T):
            r_ret = ret[sl][s * C:(s + 1) * C]
            ok = r_ret >= 0
            want[s][r_ret[ok].long()] = rows[s * C:(s + 1) * C][ok]
    for s in range(T):
        assert torch.equal(comb[s], want[s]), (s, (comb[s].float() - want[s].float()).abs().max())


# ------------------------------------------------------------------------------------------------ FusedExpertLayer
def _run_fused_layer(rank, world_size, port, top_k, capacity, gate_scale, ns):
    from pipegoose_b200.models.bloom import BloomConfig, BloomMLP
    from pipegoose_b200.nn.expert_parallel import ExpertContext, Top1Router, Top2Router
    from pipegoose_b200.ops import kernels as K_
    from pipegoose_b200.ops.moe import FusedExpertLayer
    from pipegoose_b200.testing.utils import init_parallel_context

    ctx = init_parallel_context(rank, world_size, port, world_size, 1, 1, backend="nccl")
    dev = torch.device("cuda", torch.cuda.current_device())
    E, h, alpha = 6, 256, 0.01
    torch.manual_seed(0)
    expert = BloomMLP(BloomConfig(hidden_size=h, n_head=4))
    router = (Top1Router if top_k == 1 else Top2Router)(None, E, h, expert_capacity=capacity, alpha=alpha)
    layer = FusedExpertLayer(E, expert, router, ctx).to(torch.bfloat16).to(dev)
    g = torch.Generator().manual_seed(5)
    W1 = (torch.randn(E, 4 * h, h, generator=g) * 0.05).to(torch.bfloat16)
    B1 = (torch.randn(E, 4 * h, generator=g) * 0.05).to(torch.bfloat16)
    W2 = (torch.randn(E, h, 4 * h, generator=g) * 0.05).to(torch.bfloat16)
    B2 = (torch.randn(E, h, generator=g) * 0.05).to(torch.bfloat16)
    Wg = (torch.randn(E, h, generator=g) * gate_scale).to(torch.bfloat16)
    Bg = (torch.randn(E, generator=g) * 0.5).to(torch.bfloat16)
    drops = capacity[0] < 1.0
    with torch.no_grad():
        layer.w1.copy_(W1); layer.b1.copy_(B1); layer.w2.copy_(W2); layer.b2.copy_(B2)
        layer.router.gate.weight.copy_(Wg); layer.router.gate.bias.copy_(Bg)
    layer.eval()
    ectx = ExpertContext.get_instance()

    def rel(a, b):
        return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)

    W1f, B1f, W2f, B2f, Wgf, Bgf = (t.float().to(dev).requires_grad_(True) for t in (W1, B1, W2, B2, Wg, Bg))
    for n in ns:                      # two token counts: two workspaces
        X = torch.randn(n, h, generator=g).to(torch.bfloat16).to(dev)
        Rs = torch.randn(n, h, generator=g).to(torch.bfloat16).to(dev) if not drops else torch.zeros(n, h, dtype=torch.bfloat16, device=dev)
        DY = torch.randn(n, h, generator=g).to(torch.bfloat16).to(dev)
        # dense fp32 reference over all experts
        Xf = X.float().requires_grad_(True)
        logits = Xf @ Wgf.t() + Bgf
        probs = torch.softmax(logits, dim=-1)
        tp, ti = torch.topk(probs, top_k, dim=-1)
        he = torch.stack([K_.gelu_tanh(Xf @ W1f[e].t() + B1f[e]) @ W2f[e].t() + B2f[e] for e in range(E)], 1)  # [n, E, h]
        mask = torch.zeros(n, E, device=dev).scatter_(1, ti, 1.0)
        want_aux = alpha * E * torch.dot(mask.mean(0), probs.mean(0)).item()
        want_z = torch.logsumexp(logits, -1).square().mean().item()
        for call in range(2):         # two calls: both buffer parities, forward and backward
            for p in layer.parameters():
                p.grad = None
            ectx.pop_all_aux_loss(); ectx.pop_all_z_loss()
            x = X.clone().requires_grad_(True)
            res = Rs.clone().requires_grad_(True)
            y = layer(x, res)
            aux, zl = ectx.pop_all_aux_loss(), ectx.pop_all_z_loss()
            assert len(aux) == 1 and len(zl) == 1
            assert abs(aux[0].item() - want_aux) <= 1e-3 * abs(want_aux), (aux[0].item(), want_aux)
            assert abs(zl[0].item() - want_z) <= 1e-3 * abs(want_z), (zl[0].item(), want_z)
            if not drops:
                out = Rs.float() + (tp.unsqueeze(-1) * he.gather(1, ti.unsqueeze(-1).expand(n, top_k, h))).sum(1)
                assert rel(y, out) < 3e-2, (n, call, rel(y, out))
                y.backward(DY)
                for t in (Xf, W1f, B1f, W2f, B2f, Wgf, Bgf):
                    t.grad = None
                out.backward(DY.float(), retain_graph=True)
                assert rel(x.grad, Xf.grad) < 6e-2, rel(x.grad, Xf.grad)
                assert torch.equal(res.grad, DY)
                assert rel(layer.w1.grad, W1f.grad) < 6e-2 and rel(layer.w2.grad, W2f.grad) < 6e-2
                assert rel(layer.b1.grad, B1f.grad) < 6e-2 and rel(layer.b2.grad, B2f.grad) < 6e-2
                assert rel(layer.router.gate.weight.grad, Wgf.grad) < 1e-1
                assert rel(layer.router.gate.bias.grad, Bgf.grad) < 1e-1
                continue
            # capacity-limited (zero residual): every row is sum_{kept k} p_k expert_k(x) for SOME kept subset, and
            # the number kept per expert is min(count, C)
            with torch.no_grad():
                terms = tp.unsqueeze(-1) * he.gather(1, ti.unsqueeze(-1).expand(n, top_k, h))   # [n, K, h]
                subsets = torch.tensor(list(itertools.product([0.0, 1.0], repeat=top_k)), device=dev)  # [S, K]
                cands = torch.einsum("sk,nkh->nsh", subsets, terms)
                err = (y.float().unsqueeze(1) - cands).norm(dim=-1)                      # [n, S]
                best = err.argmin(1)
                scale = cands.norm(dim=-1).max(1).values.clamp_min(1e-3)
                assert bool((err.gather(1, best[:, None])[:, 0] <= 3e-2 * scale).all()), (err.min(1).values / scale).max()
                kept = subsets[best]                                                     # [n, K]
                C = layer._workspace(n, h).C
                counts = torch.bincount(ti.flatten(), minlength=E)
                kept_per_e = torch.zeros(E, device=dev).scatter_add_(0, ti.flatten(), kept.flatten())
                assert torch.equal(kept_per_e.long(), counts.clamp(max=C)), (kept_per_e, counts, C)
                assert bool((counts > C).any()), "no token was dropped"
    torch.cuda.synchronize()
    ctx.destroy()


@pytest.mark.parametrize("top_k", [1, 2])
def test_fused_expert_layer_single_gpu(top_k):
    """``FusedExpertLayer`` in a one-rank group (T = 1): forward, backward and the pushed router losses against the
    dense fp32 reference, over two calls (both buffer parities) at two token counts (two workspaces)."""
    from pipegoose_b200.testing.utils import spawn

    spawn(_run_fused_layer, world_size=1, top_k=top_k, capacity=(8.0, 8.0), gate_scale=0.5, ns=(512, 384))


@pytest.mark.parametrize("top_k", [1, 2])
def test_fused_expert_layer_capacity_drops(top_k):
    """``expert_capacity = (0.5, 0.5)``: tokens over an expert's capacity are dropped, whichever they are.  A flatter
    gate keeps every chosen expert's weight large enough to tell which terms a row kept."""
    from pipegoose_b200.testing.utils import spawn

    spawn(_run_fused_layer, world_size=1, top_k=top_k, capacity=(0.5, 0.5), gate_scale=0.05, ns=(1024,))
