"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op (GPU only)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _native():
    from pipegoose_b200 import ops

    return ops.native()


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
@pytest.mark.parametrize("shape", [(512, 384, 256), (1000, 264, 200), (2048, 1024, 1024)])
def test_gemm_layouts(layout, shape):
    from pipegoose_b200.ops import kernels as K

    M, N, Kd = shape
    torch.manual_seed(0)
    if layout == "nt":
        x = torch.randn(M, Kd, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, Kd, device="cuda", dtype=torch.bfloat16)
        out, ref = K.gemm_nt(x, w), x.float() @ w.float().t()
    elif layout == "nn":
        dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, Kd, device="cuda", dtype=torch.bfloat16)
        out, ref = K.gemm_nn(dy, w), dy.float() @ w.float()
    else:
        if M % 8:
            pytest.skip("wgrad needs 16B-aligned rows")
        dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
        x = torch.randn(M, Kd, device="cuda", dtype=torch.bfloat16)
        out, ref = K.gemm_tn(dy, x), dy.float().t() @ x.float()
    assert _rel(out, ref) < 1e-2


def test_gemm_epilogues():
    from pipegoose_b200.ops import kernels as K

    torch.manual_seed(1)
    M, N, Kd = 640, 328, 136
    x = torch.randn(M, Kd, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(N, Kd, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, device="cuda", dtype=torch.bfloat16)
    r = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    base = x.float() @ w.float().t() + b.float()
    assert _rel(K.gemm_nt(x, w, b, r), base + r.float()) < 1e-2
    z = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    y = K.gemm_nt(x, w, b, gelu=True, aux_out=z)
    assert _rel(z, base) < 1e-2 and _rel(y, K.gelu_tanh(base)) < 1e-2
    dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    zz = torch.randn(M, Kd, device="cuda", dtype=torch.bfloat16)
    got = K.gemm_nn(dy, w, dgelu_aux=zz)
    assert _rel(got, (dy.float() @ w.float()) * K.gelu_tanh_grad(zz.float())) < 1e-2
    acc = torch.randn(N, Kd, device="cuda", dtype=torch.float32)
    want = acc + dy.float().t() @ x.float()
    K.gemm_tn(dy, x, accum_into=acc)
    assert _rel(acc, want) < 1e-3
    K.gemm_tn(dy, x, accum_into=acc, accumulate=False)
    assert _rel(acc, dy.float().t() @ x.float()) < 1e-3


@pytest.mark.parametrize("h", [64, 1024, 2560, 4096])
def test_layernorm(h):
    from pipegoose_b200.ops import kernels as K

    torch.manual_seed(2)
    rows = 777
    x = torch.randn(rows, h, device="cuda", dtype=torch.bfloat16) * 2 + 0.5
    g = torch.randn(h, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(h, device="cuda", dtype=torch.bfloat16)
    y, mean, rstd = K.layernorm_fwd(x, g, b, 1e-5)
    xf = x.float().requires_grad_(True)
    gf, bf = g.float().requires_grad_(True), b.float().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xf, (h,), gf, bf, 1e-5)
    assert _rel(y, ref) < 1e-2
    dy = torch.randn(rows, h, device="cuda", dtype=torch.bfloat16)
    extra = torch.randn(rows, h, device="cuda", dtype=torch.bfloat16)
    ref.backward(dy.float())
    dx, dg, db = K.layernorm_bwd(dy, x, g, mean, rstd, dx_extra=extra)
    assert _rel(dx, xf.grad + extra.float()) < 2e-2
    assert _rel(dg, gf.grad) < 2e-2 and _rel(db, bf.grad) < 2e-2


def test_embedding_and_colsum():
    from pipegoose_b200.ops import kernels as K

    torch.manual_seed(3)
    V, h, rows = 1000, 256, 513
    table = torch.randn(V, h, device="cuda", dtype=torch.bfloat16)
    g = torch.ones(h, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros(h, device="cuda", dtype=torch.bfloat16)
    ids = torch.randint(0, 2 * V, (rows,), device="cuda")
    e, _, _ = K.layernorm_fwd(table, g, b, 1e-5, ids=ids, vocab_start=V // 2, vocab_end=V // 2 + V, apply_ln=False)
    mask = (ids >= V // 2) & (ids < V // 2 + V)
    ref = table[(ids - V // 2).clamp(0, V - 1)] * mask[:, None]
    assert torch.equal(e, ref)
    dx = torch.randn(rows, h, device="cuda", dtype=torch.bfloat16)
    dw = K.embedding_bwd(dx, ids, V, V // 2, V // 2 + V)
    want = torch.zeros(V, h, device="cuda")
    want.index_add_(0, (ids - V // 2)[mask], dx.float()[mask])
    assert _rel(dw, want) < 1e-2
    assert _rel(K.colsum(dx), dx.float().sum(0)) < 1e-2


@pytest.mark.parametrize("V", [1000, 32768 + 8])
def test_cross_entropy(V):
    from pipegoose_b200.ops import kernels as K

    torch.manual_seed(4)
    rows = 300
    logits = (torch.randn(rows, V, device="cuda") * 3).to(torch.bfloat16)
    tgt = torch.randint(0, V, (rows,), device="cuda")
    tgt[::7] = -100
    lf = logits.float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf, tgt, ignore_index=-100, reduction="sum")
    ref.backward()
    stats = K.ce_local_stats(logits, tgt, 0)
    work = logits.clone()
    scale = torch.tensor([0.5], device="cuda")
    loss_rows = K.ce_finalize(work, tgt, stats, 0, scale, -100, write_grad=True)
    assert abs(loss_rows.sum().item() - ref.item()) / abs(ref.item()) < 1e-3
    assert _rel(work, lf.grad * 0.5) < 2e-2


def test_fused_adam_matches_torch():
    from pipegoose_b200.ops import kernels as K  # noqa: F401

    torch.manual_seed(5)
    n = 100003
    p = torch.randn(n, device="cuda")
    ref_p = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref_p], lr=1e-2)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    pb = p.to(torch.bfloat16)
    for step in range(1, 4):
        g = torch.randn(n, device="cuda")
        ref_p.grad = g.clone()
        opt.step()
        _native().adam_step(p, m, v, g, pb, 1e-2, 0.9, 0.999, 1e-8, 0.0, step, 1.0, False)
    assert _rel(p, ref_p.detach()) < 1e-5
    assert _rel(pb, ref_p.detach()) < 1e-2


def test_bloom_matches_fp32_reference():
    """Fused bf16 Bloom (GPU kernels) vs the same model evaluated in fp32 with PyTorch ops on the CPU."""
    import copy

    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM

    torch.manual_seed(6)
    cfg = BloomConfig(vocab_size=4096, hidden_size=256, n_layer=2, n_head=4)
    ref = BloomForCausalLM(cfg)
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if "layernorm" in n or "ln_f" in n or "bias" in n:
                p.add_(torch.randn_like(p) * 0.1)
    model = copy.deepcopy(ref).to(torch.bfloat16).cuda()
    # evaluate the reference at the bf16-rounded weights
    ref.load_state_dict({k: v.float().cpu() for k, v in model.state_dict().items()})
    ids = torch.randint(0, cfg.vocab_size, (2, 256))
    lr = ref(ids, labels=ids).loss
    lr.backward()
    lg = model(ids.cuda(), labels=ids.cuda()).loss
    lg.backward()
    assert abs(lg.item() - lr.item()) < 3e-2
    logits_g = model(ids.cuda()).logits
    logits_r = ref(ids).logits
    assert _rel(logits_g.cpu(), logits_r) < 3e-2
    rp = dict(ref.named_parameters())
    bad = []
    for n, p in model.named_parameters():
        r = _rel(p.grad.cpu(), rp[n].grad)
        if r > 8e-2:
            bad.append((n, r))
    assert not bad, bad


@pytest.mark.parametrize("D,H,S,B", [(64, 4, 512, 2), (64, 16, 1024, 2), (128, 2, 384, 1), (128, 4, 1024, 2)])
def test_flash_alibi_attention(D, H, S, B):
    from pipegoose_b200.ops import kernels as K
    from pipegoose_b200.ops.attention import _AlibiAttentionNative, alibi_attention_reference

    torch.manual_seed(7)
    qkv = torch.randn(B * S, H * 3 * D, device="cuda", dtype=torch.bfloat16)
    slopes = K.alibi_slopes(H, device="cuda")
    qkv_g = qkv.clone().requires_grad_(True)
    out = _AlibiAttentionNative.apply(qkv_g, slopes, B, S, H, D)
    ref_in = qkv.float().requires_grad_(True)
    ref = alibi_attention_reference(ref_in, slopes, B, S, H, D)
    assert _rel(out, ref) < 2e-2
    dout = torch.randn_like(out)
    out.backward(dout)
    ref.backward(dout.float())
    g, r = qkv_g.grad.view(B * S, H, 3, D).float(), ref_in.grad.view(B * S, H, 3, D)
    for i, name in enumerate("qkv"):
        assert _rel(g[:, :, i], r[:, :, i]) < 3e-2, name


@pytest.mark.parametrize("M,V,valid", [(512, 4096, 4096), (384, 1000, 1000), (256, 2560, 2500)])
def test_lm_head_ce_stats_in_epilogue(M, V, valid):
    """The logits GEMM epilogue's online-softmax partials, merged by ce_combine, equal the statistics of a pass over the
    stored logits (exactly the same bf16 values) — also with vocabulary padding and a last partial tile."""
    from pipegoose_b200.ops import kernels as K

    torch.manual_seed(0)
    x = (torch.randn(M, 256, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(V, 256, device="cuda") * 0.2).to(torch.bfloat16)
    tgt = torch.randint(0, valid, (M,), device="cuda")
    part = K.ce_partials_buffer(M, V, x.device)
    part.fill_(float("nan"))
    logits = K.gemm_nt(x, w, ag={"ce_part": part.data_ptr(), "ce_valid": valid})
    plain = K.gemm_nt(x, w)
    assert torch.equal(logits, plain)
    assert not torch.isnan(part).any(), "a (row, tile, half) slot was not written"
    if valid < V:
        logits[:, valid:] = float("-inf")
    got = K.ce_stats_from_partials(part, logits, tgt, 0)
    want = K.ce_local_stats(logits, tgt, 0)
    lse_got = got[:, 0] + torch.log(got[:, 1])
    lse_want = want[:, 0] + torch.log(want[:, 1])
    assert torch.allclose(lse_got, lse_want, atol=1e-4, rtol=1e-5), (lse_got - lse_want).abs().max()
    assert torch.equal(got[:, 2], want[:, 2])


def test_lm_head_cross_entropy_with_epilogue_stats_matches(monkeypatch):
    """LMHeadCrossEntropy with the statistics taken from the GEMM epilogue: same loss and gradients."""
    from pipegoose_b200.ops import functional as PF

    torch.manual_seed(1)
    h, V, M = 256, 4096, 512
    x = (torch.randn(M, h, device="cuda") * 0.5).to(torch.bfloat16)
    gamma = torch.ones(h, device="cuda", dtype=torch.bfloat16)
    beta = torch.zeros(h, device="cuda", dtype=torch.bfloat16)
    table = (torch.randn(V, h, device="cuda") * 0.05).to(torch.bfloat16)
    labels = torch.randint(0, V, (M,), device="cuda")
    out = {}
    for name, flag in (("pass", False), ("epilogue", True)):
        monkeypatch.setattr(PF, "_CE_IN_EPILOGUE", flag)
        xi, ti = x.clone().requires_grad_(True), table.clone().requires_grad_(True)
        loss = PF.lm_head_cross_entropy(xi, gamma, beta, ti, labels)
        loss.backward()
        out[name] = (loss.item(), xi.grad.float(), ti.grad.float())
    assert abs(out["pass"][0] - out["epilogue"][0]) < 1e-5
    assert torch.allclose(out["pass"][1], out["epilogue"][1], atol=1e-5, rtol=1e-3)
    assert torch.allclose(out["pass"][2], out["epilogue"][2], atol=1e-5, rtol=1e-3)


def test_vocab_parallel_cross_entropy_backward_uses_the_kernel():
    """The reference-compatible VocabParallelCrossEntropy (class-swap path): bf16 CUDA logits take the fused finalize
    kernel in backward; loss and gradient match torch's cross entropy."""
    from pipegoose_b200.nn.tensor_parallel.loss import VocabParallelCrossEntropy

    class OneRank:
        def get_world_size(self, mode):
            return 1

        def get_local_rank(self, mode):
            return 0

    torch.manual_seed(3)
    B, S, V = 4, 64, 4096
    logits = (torch.randn(B, S, V, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    tgt = torch.randint(0, V, (B, S), device="cuda")
    loss = VocabParallelCrossEntropy(OneRank())(logits, tgt)
    loss.backward()
    ref_in = logits.detach().float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(ref_in.view(-1, V), tgt.view(-1))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 2e-3
    assert _rel(logits.grad.float(), ref_in.grad) < 2e-2
