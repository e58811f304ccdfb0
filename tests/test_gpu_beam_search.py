"""Beam search on the GPU: ``beam_topk_kernel`` against a float64 reference with a derived error bound,
``paged_kv_copy_kernel`` against its reference bit for bit, and ``ContinuousBatcher`` beam requests on bf16 Bloom and
GPT-2 in every serving mode, against the training forward and against 🤗 fp32 beam search.

Bound of a reported score.  The kernel computes ``s = b + (x - lse)`` in fp32 from the same bf16 / fp32 logits x the
float64 reference reads, with ``lse = m + log(sum)``.  The sum has at most ``L = ceil(V / 256) + 64`` sequential
steps per thread, warp, CTA and split merge, each adding one fp32 rounding (2^-24 relative) and, where it rescales,
one ``__expf`` error of at most 4 * 2^-24 relative for the arguments that matter (``x - m`` near 0; terms far below
the maximum carry their error in proportion to their size).  So the relative error of the sum, and the absolute error
of its log, is at most ``5 L 2^-24``; ``logf`` adds 2 ulp of lse, and the two fp32 operations of ``s`` one ulp each of
``|x - lse|`` and ``|s|``.  ``bound = 6 L 2^-24 + (2 |lse| + |x - lse| + |s| + 1) 2^-23``."""
import copy
import math

import pytest
import torch

from pipegoose_b200.ops.attention import PAGE_SIZE, paged_kv_copy, paged_kv_copy_reference, quantize_kv
from pipegoose_b200.ops.kernels import beam_topk
from pipegoose_b200.serving import ContinuousBatcher

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn


def _inputs(V, rows, dtype, strided, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N = sum(rows)
    width = V + 40 if strided else V
    base = torch.randn(N, width, generator=g, device="cuda") * 4
    logits = base[:, 5:5 + V] if strided else base
    if V > 8:
        logits[:, V // 3] = float("-inf")                          # vocabulary padding columns
        logits[:, -1] = float("-inf")
    logits[0] = 1.5                                                # a row of equal logits
    if V > 8:
        logits[0, V // 3] = float("-inf")
    logits = logits.to(dtype)
    scores = torch.randn(N, generator=g, device="cuda") * 3
    cu = [0]
    for n in rows:
        cu.append(cu[-1] + n)
    for r, (a, b) in enumerate(zip(cu, cu[1:])):
        if r % 2:
            scores[a + 1:b] = -1e9                                 # 🤗's first step: one live beam
    return logits, scores, cu


def _bound(x64, lse64, s64, V):
    L = math.ceil(V / 256) + 64
    return 6 * L * 2 ** -24 + (2 * lse64.abs() + (x64 - lse64).abs() + s64.abs() + 1) * 2 ** -23


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("V,rows,k,strided", [
    (7, [1, 2, 3], 6, False),
    (1000, [1, 8, 3, 4, 2, 5, 7, 6], 16, True),
    (50257, [2] * 16 + [1] * 8, 4, False),
    (50257, [8] * 32, 16, True),
    (250880, [1], 2, False),
    (250880, [4, 2, 8, 1], 16, False),
    (250880, [8] * 32, 16, False),
])
def test_beam_topk_kernel_against_float64(V, rows, k, strided, dtype):
    logits, scores, cu = _inputs(V, rows, dtype, strided, seed=V + k)
    got_s, got_t, got_r, lse = beam_topk(logits, scores, cu, k, return_lse=True)
    again = beam_topk(logits, scores, cu, k, return_lse=True)
    for a, b in zip((got_s, got_t, got_r, lse), again):            # bitwise reproducible
        assert torch.equal(a, b)
    x = logits.double()
    lse64 = torch.logsumexp(x, -1)
    fin = torch.isfinite(lse64)
    assert ((lse.double() - lse64).abs()[fin] <= _bound(0 * lse64, lse64, lse64, V)[fin]).all()
    exact = x - lse64.view(-1, 1) + scores.double().view(-1, 1)
    worst = 0.0
    for r, (a, b) in enumerate(zip(cu, cu[1:])):
        flat = exact[a:b].reshape(-1)
        kth = torch.sort(flat, descending=True, stable=True).values[k - 1]
        rows_r, toks = got_r[r].long(), got_t[r].long()
        assert ((rows_r >= a) & (rows_r < b)).all() and len(set(zip(rows_r.tolist(), toks.tolist()))) == k
        want = exact[rows_r, toks]
        s = got_s[r].double()
        assert (s[1:] <= s[:-1]).all()                             # descending
        bound = _bound(x[rows_r, toks], lse64[rows_r], want, V)
        finite = torch.isfinite(want)
        assert torch.equal(finite, torch.isfinite(s))
        err = (s - want).abs()[finite]
        assert (err <= bound[finite]).all(), (r, err.max().item())
        worst = max(worst, (err / bound[finite]).max().item() if finite.any() else 0.0)
        if torch.isfinite(kth):                                    # a valid top-k under the bound
            assert (want[finite] >= kth - 2 * bound[finite]).all()
    # the row of equal logits (request 0, row 0): equal scores go to the lower token
    if rows[0] == 1:
        toks = [t for t in range(V) if not (V > 8 and t == V // 3)][:k]
        assert got_t[0].tolist() == toks and got_r[0].tolist() == [0] * k
    print(f"\nbeam_topk V={V} rows={sum(rows)} k={k} {dtype}: worst |err| / bound {worst:.3f}")


def test_beam_topk_ties_across_rows():
    """Equal rows with equal scores: the lower row first, then the lower token."""
    V = 3000
    row = torch.randn(V, device="cuda").to(torch.bfloat16)
    logits = row.view(1, V).repeat(4, 1)
    scores = torch.zeros(4, device="cuda")
    s, t, r, _ = beam_topk(logits, scores, [0, 4], 16)
    vals = row.float().tolist()
    want = [(n, tok) for _, n, tok in sorted((-vals[tok], n, tok) for n in range(4) for tok in range(V))[:16]]
    assert list(zip(r[0].tolist(), t[0].tolist())) == want


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_kv_copy_kernel_is_the_reference(D, fp8):
    L, pages, H = 3, 9, 4                   # page 8 plays the graphs' scratch page
    k = torch.full((L, pages, H, PAGE_SIZE, D), float("nan"), device="cuda")
    v = torch.full_like(k, float("nan"))
    g = torch.Generator(device="cuda").manual_seed(D)
    k[:, :5] = torch.randn(L, 5, H, PAGE_SIZE, D, generator=g, device="cuda")
    v[:, :5] = torch.randn(L, 5, H, PAGE_SIZE, D, generator=g, device="cuda")
    ks = vs = None
    if fp8:
        (k, ks), (v, vs) = quantize_kv(k), quantize_kv(v)
    else:
        k, v = k.to(torch.bfloat16), v.to(torch.bfloat16)
    pairs = [[(0, 5, 0), (1, 6, 1), (2, 7, 63), (3, 8, 64)], [(8, 4, 17)]]     # into, then out of, the scratch page
    cpu = [t.cpu() if t is not None else None for t in (k, v, ks, vs)]

    def bits(t):
        return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int16) if t.element_size() == 2 else t.view(
            torch.int32)
    for p in pairs:
        paged_kv_copy(p, k, v, ks, vs)
        paged_kv_copy_reference(p, *cpu)
    for a, b in zip((k, v, ks, vs), cpu):
        if a is not None:
            assert torch.equal(bits(a.cpu()), bits(b))


# ------------------------------------------------------------------------------------------------------- the engine
def _model(arch, hidden, n_head, ln_gain=1.0):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    if arch == "bloom":
        model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head))
    else:
        model = GPT2LMHeadModel(GPT2Config(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head,
                                           n_positions=512))
    with torch.no_grad():
        model.transformer.ln_f.weight.mul_(ln_gain)
    return model


_MODES = {"default": {}, "prefix": {"prefix_caching": True}, "fp8": {"kv_cache_dtype": FP8},
          "chunked": {"chunked_prefill": True, "max_prefill_tokens": 128}, "graphs": {"cuda_graphs": True},
          "fp8_chunked_graphs": {"kv_cache_dtype": FP8, "chunked_prefill": True, "max_prefill_tokens": 128,
                                 "cuda_graphs": True}}
_REQS = [   # (prompt length, max_new_tokens, W, length_penalty, early_stopping)
    (130, 20, 4, 1.0, False), (63, 40, 2, 0.0, "never"), (64, 12, 8, 2.0, True), (1, 30, 3, -0.5, False)]


def _serve(model, kw, prompts, greedy):
    engine = ContinuousBatcher(model, max_cache_tokens=96 * PAGE_SIZE, **kw)
    rids = [engine.submit(p, n, num_beams=W, length_penalty=lp, early_stopping=es, num_return_sequences=W)
            for p, (_, n, W, lp, es) in zip(prompts, _REQS)]
    gids = [engine.submit(p, 25) for p in greedy]
    outs = engine.run()
    assert len(engine._free) == engine.num_pages and engine.beam_page_copies > 0
    return [engine.hypotheses.pop(r) for r in rids], [outs[g] for g in gids], outs, rids


@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_engine_scores_match_the_training_forward(arch, hidden, n_head):
    model = _model(arch, hidden, n_head).to(torch.bfloat16).cuda().eval()
    g = torch.Generator().manual_seed(hidden)
    prompts = [torch.randint(0, 4096, (P,), generator=g).tolist() for P, *_ in _REQS]
    greedy = [torch.randint(0, 4096, (n,), generator=g).tolist() for n in (40, 90)]
    base, base_greedy, _, _ = _serve(model, {}, prompts, greedy)
    for mode, kw in _MODES.items():
        hyps, _, outs, rids = _serve(model, kw, prompts, greedy) if mode != "default" else (base, None, None, None)
        for i, ((P, n, W, lp, es), hs) in enumerate(zip(_REQS, hyps)):
            assert len(hs) == W and all(P < len(t) <= P + n for t, _ in hs)
            if outs is not None:
                assert outs[rids[i]] == hs[0][0]
            for tokens, score in hs:
                with torch.no_grad():
                    logits = model(torch.tensor([tokens], device="cuda")).logits[0].float()
                lp_all = torch.log_softmax(logits[P - 1:-1], -1)
                gen = len(tokens) - P
                total = lp_all.gather(1, torch.tensor(tokens[P:], device="cuda").view(-1, 1)).sum().item()
                tol = 2 * gen * 3e-2 * logits[P - 1:].abs().max().item() / gen ** lp
                assert abs(score - total / gen ** lp) <= tol, (mode, i, score, total / gen ** lp, tol)
                assert score <= base[i][0][1] + tol, (mode, i)


def test_engine_tokens_match_hf_fp32_beam_search():
    """An fp32 model on the GPU (the engine then runs the PyTorch references on the device, as for every serving op):
    token for token and score for score against 🤗 fp32 beam search on the same weights, with eos reached and not.
    On random-init weights the bf16 engine's rounding is larger than the gaps between competing candidates, so its
    tokens are checked against the training forward's scores above instead."""
    model = _model("bloom", 256, 4).cuda().eval()
    hf = copy.deepcopy(model).to_hf().cuda().eval()
    g = torch.Generator().manual_seed(2)
    reqs = [(P, n, W, lp, es) for P, n in ((3, 70), (64, 20), (130, 9))
            for W, lp, es in ((2, 1.0, False), (4, 0.0, "never"), (8, 2.0, True))]
    prompts = [torch.randint(0, 4096, (P,), generator=g).tolist() for P, *_ in reqs]
    for use_eos in (False, True):
        engine = ContinuousBatcher(model, max_cache_tokens=160 * PAGE_SIZE, prefix_caching=use_eos)
        eos = [model.generate(torch.tensor([p], device="cuda"), max_new_tokens=4)[0, -1].item() if use_eos else None
               for p in prompts]
        rids = [engine.submit(p, n, num_beams=W, length_penalty=lp, early_stopping=es, num_return_sequences=W,
                              eos_token_id=e) for p, (_, n, W, lp, es), e in zip(prompts, reqs, eos)]
        engine.run()
        assert len(engine._free) == engine.num_pages
        for p, (P, n, W, lp, es), rid, e in zip(prompts, reqs, rids, eos):
            out = hf.generate(torch.tensor([p], device="cuda"), max_new_tokens=n, num_beams=W, length_penalty=lp,
                              early_stopping=es, num_return_sequences=W, eos_token_id=10 ** 6 if e is None else e,
                              pad_token_id=0, do_sample=False, return_dict_in_generate=True, output_scores=True)
            for j, (tokens, score) in enumerate(engine.hypotheses.pop(rid)):
                L = int((out.beam_indices[j] >= 0).sum())
                assert tokens == out.sequences[j, :P + L].tolist(), (P, W, j, use_eos)
                assert abs(score - out.sequences_scores[j].item()) <= 1e-4, (P, W, j, use_eos)
