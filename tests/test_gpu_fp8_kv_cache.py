"""FP8 (e4m3) paged KV cache on the GPU: the quantizing cache write bit for bit against the CPU quantizer, the FP8 split-KV
decode kernel against its fp32 reference and against the bf16 kernel, the staged cached prefill, the bindings'
refusals, and ``ContinuousBatcher(kv_cache_dtype=torch.float8_e4m3fn)`` on bf16 models against the bf16-pool engine
(teacher-forced) and the fp32 reference path over the same FP8 pools."""
import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops import native
from pipegoose_b200.ops.attention import (PAGE_SIZE, alibi_paged_decode_attention,
                                          alibi_paged_decode_attention_reference, alibi_paged_prefill_attention,
                                          alibi_paged_prefill_attention_reference, dequantize_kv, fp8_prefill_staging,
                                          paged_kv_dequantize, paged_kv_write, paged_kv_write_reference, quantize_kv)

pytestmark = pytest.mark.gpu

FP8 = torch.float8_e4m3fn
LENGTHS = [1, 2, 63, 64, 65, 1000, 4097, 33000]


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-6)


def _nan_pools(num_pages, H, D):
    """Pools of NaN codes (0x7F) and NaN scales, on the CPU."""
    k = torch.full((num_pages, H, PAGE_SIZE, D), 0x7F, dtype=torch.uint8).view(FP8)
    s = torch.full((num_pages, H, PAGE_SIZE), float("nan"))
    return k, k.clone(), s, s.clone()


def _same(a, b):
    """Bitwise equality (NaN included)."""
    view = torch.uint8 if a.dtype == FP8 else torch.int32
    return torch.equal(a.cpu().view(view), b.cpu().view(view))


def _fp8_case(H, D, lengths, seed, spare_pages=5, filled=None):
    """NaN pools with quantized random keys / values in every row's first ``filled[b]`` positions (default: all but
    the last) and a shuffled page table; all on the CPU."""
    g = torch.Generator().manual_seed(seed)
    filled = filled or [n - 1 for n in lengths]
    need = [(n - 1) // PAGE_SIZE + 1 for n in lengths]
    num_pages = sum(need) + spare_pages
    perm = torch.randperm(num_pages, generator=g).to(torch.int32)
    table = torch.full((len(lengths), max(need) + 1), -7, dtype=torch.int32)   # never read
    k_pool, v_pool, k_scales, v_scales = _nan_pools(num_pages, H, D)
    used = 0
    for b, n in enumerate(lengths):
        table[b, :need[b]] = perm[used:used + need[b]]
        used += need[b]
        p = torch.arange(filled[b])
        pages, slots = table[b, p // PAGE_SIZE].long(), p % PAGE_SIZE
        for pool, scales in ((k_pool, k_scales), (v_pool, v_scales)):
            codes, s = quantize_kv(torch.randn(filled[b], H, D, generator=g).to(torch.bfloat16))
            pool[pages, :, slots], scales[pages, :, slots] = codes, s
    return k_pool, v_pool, k_scales, v_scales, table


@pytest.mark.parametrize("D", [64, 80, 128])
def test_fp8_cache_write_is_bitwise_the_quantizer(D):
    H, N = 3, 200
    g = torch.Generator().manual_seed(D)
    qkv = torch.randn(N, H, 3, D, generator=g)
    qkv[5, :, 1] = 0.0                                     # zero rows
    qkv[6, 1, 2] = -0.0
    qkv[7, 0, 1, 3] = 3e4                                  # one large outlier
    qkv[8, 2, 2, D - 1] = -1e-30
    qkv = qkv.view(N, -1).to(torch.bfloat16)
    num_pages = 9
    slot = torch.randperm(num_pages * PAGE_SIZE, generator=g)[:N].to(torch.int32)
    k_pool, v_pool, k_scales, v_scales = _nan_pools(num_pages, H, D)
    paged_kv_write_reference(qkv, slot, k_pool, v_pool, D, k_scales, v_scales)
    gpu = [t.cuda() for t in _nan_pools(num_pages, H, D)]
    paged_kv_write(qkv.cuda(), slot.cuda(), gpu[0], gpu[1], D, k_scales=gpu[2], v_scales=gpu[3])
    for want, got in zip((k_pool, v_pool, k_scales, v_scales), gpu):
        assert _same(got, want)
    assert (k_scales[slot // PAGE_SIZE, :, slot % PAGE_SIZE] == 0).sum() >= H


@pytest.mark.parametrize("D", [64, 80, 128])
def test_fp8_decode_kernel_matches_reference(D):
    H = 2
    lengths = LENGTHS[D % 3:] + LENGTHS[:D % 3]
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, lengths, seed=D)
    g = torch.Generator().manual_seed(D + 1)
    qkv = torch.randn(len(lengths), H * 3 * D, generator=g).to(torch.bfloat16)
    pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32)
    slopes = K.alibi_slopes(H)
    max_pos = max(lengths) - 1
    gpu = [t.cuda() for t in (k_pool, v_pool, k_scales, v_scales)]
    out = alibi_paged_decode_attention(qkv.cuda(), gpu[0], gpu[1], table.cuda(), pos.cuda(), max_pos,
                                       slopes.cuda(), D, k_scales=gpu[2], v_scales=gpu[3])
    ref = alibi_paged_decode_attention_reference(qkv.float(), k_pool, v_pool, table, pos, max_pos, slopes, D,
                                                 k_scales=k_scales, v_scales=v_scales)
    assert torch.isfinite(out).all()
    for b in range(len(lengths)):
        assert _rel(out[b], ref[b]) < 1e-2, lengths[b]
    # the reference stored every pos[b] slot with the quantizer; nothing else changed on either side
    for want, got in zip((k_pool, v_pool, k_scales, v_scales), gpu):
        assert _same(got, want)
    again = alibi_paged_decode_attention(qkv.cuda(), gpu[0], gpu[1], table.cuda(), pos.cuda(), max_pos,
                                         slopes.cuda(), D, k_scales=gpu[2], v_scales=gpu[3])
    assert torch.equal(out, again)
    loose = alibi_paged_decode_attention(qkv.cuda(), gpu[0], gpu[1], table.cuda(), pos.cuda(),
                                         table.shape[1] * PAGE_SIZE - 1, slopes.cuda(), D, k_scales=gpu[2],
                                         v_scales=gpu[3])
    assert torch.isfinite(loose).all() and _rel(loose, out) < 1e-2


@pytest.mark.parametrize("D", [64, 80, 128])
def test_fp8_decode_kernel_equals_bf16_kernel_on_exact_values(D):
    """Power-of-two scales: every dequantized value is exact in bf16, so the bf16 kernel on the dequantized pools does
    the same arithmetic up to fp32 summation order (and one bf16 rounding of the output)."""
    H = 4
    lengths = [1, 100, 3000, 9000]
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, lengths, seed=D + 2)
    g = torch.Generator().manual_seed(D + 3)
    for scales in (k_scales, v_scales):
        finite = scales.isfinite()
        scales[finite] = 2.0 ** torch.randint(-6, -3, (int(finite.sum()),), generator=g).float()
    k16 = dequantize_kv(k_pool, k_scales).to(torch.bfloat16).cuda()
    v16 = dequantize_kv(v_pool, v_scales).to(torch.bfloat16).cuda()
    qkv = torch.randn(len(lengths), H * 3 * D, generator=g).to(torch.bfloat16).cuda()
    pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32, device="cuda")
    slopes = K.alibi_slopes(H, device="cuda")
    gpu = [t.cuda() for t in (k_pool, v_pool, k_scales, v_scales)]
    got = alibi_paged_decode_attention(qkv, gpu[0], gpu[1], table.cuda(), pos, max(lengths) - 1, slopes, D,
                                       k_scales=gpu[2], v_scales=gpu[3]).float()
    want = alibi_paged_decode_attention(qkv, k16, v16, table.cuda(), pos, max(lengths) - 1, slopes, D).float()
    assert ((got - want).abs() <= 2.0 ** -7 * want.abs() + 1e-4).all(), (got - want).abs().max().item()


# (starts, news) of the cached prefill: prefixes of 0, 1, 16, 65 and 2 pages; then two cases with 8192-position
# prefixes next to short ones and new tokens crossing block boundaries
PREFILL_CASES = [([0, 64, 1024, 4160, 128], [129, 1, 1000, 127, 128]),
                 ([0, 64, 192, 8192], [129, 1, 1000, 300]),
                 ([8192, 0, 640, 64, 128], [64, 127, 128, 513, 1])]


@pytest.mark.parametrize("D,starts,news", [pytest.param(D, s, n, id=f"{D}-long{i}" if i else f"{D}")
                                           for i, (s, n) in enumerate(PREFILL_CASES) for D in (64, 80, 128)])
def test_fp8_cached_prefill_matches_reference(D, starts, news):
    H = 2
    lengths = [s + n for s, n in zip(starts, news)]
    k_pool, v_pool, k_scales, v_scales, table = _fp8_case(H, D, lengths, seed=D + 4, filled=starts)
    g = torch.Generator().manual_seed(D + 5)
    qkv = torch.randn(sum(news), H * 3 * D, generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32)
    start = torch.tensor(starts, dtype=torch.int32)
    slopes = K.alibi_slopes(H)
    pages = [table[r, :(n - 1) // PAGE_SIZE + 1].tolist() for r, n in enumerate(lengths)]
    n, src, dst, slot, st_table = fp8_prefill_staging(pages, starts, lengths)
    gpu = [t.cuda() for t in (k_pool, v_pool, k_scales, v_scales)]
    k_stage = torch.full((n, H, PAGE_SIZE, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    v_stage = k_stage.clone()
    dev = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
    stage = (k_stage, v_stage, dev(src), dev(dst), dev(slot), dev(st_table))
    got = alibi_paged_prefill_attention(qkv.cuda(), gpu[0], gpu[1], table.cuda(), cu.cuda(), start.cuda(),
                                        max(news), slopes.cuda(), D, k_scales=gpu[2], v_scales=gpu[3], stage=stage)
    want = alibi_paged_prefill_attention_reference(qkv.float(), k_pool, v_pool, table, cu, start, max(news), slopes,
                                                   D, k_scales=k_scales, v_scales=v_scales)
    assert torch.isfinite(got).all()
    for r in range(len(starts)):
        assert _rel(got[cu[r]:cu[r + 1]], want[cu[r]:cu[r + 1]]) < 1e-2, (starts[r], news[r])
    # the staging pool: dequantized cached pages, bit for bit as the reference rounds them to bf16
    for s, d in zip(src, dst):
        assert torch.equal(k_stage[d].cpu(), dequantize_kv(k_pool[s], k_scales[s]).to(torch.bfloat16))
        assert torch.equal(v_stage[d].cpu(), dequantize_kv(v_pool[s], v_scales[s]).to(torch.bfloat16))
    for want_t, got_t in zip((k_pool, v_pool, k_scales, v_scales), gpu):   # the op does not write the FP8 pools
        assert _same(got_t, want_t)
    k_again = torch.empty_like(k_stage)
    paged_kv_dequantize(gpu[0], gpu[1], gpu[2], gpu[3], dev(src), dev(dst), k_again, torch.empty_like(v_stage))
    assert torch.equal(k_again[dev(dst).long()], k_stage[dev(dst).long()])


def test_fp8_refusals():
    H, D = 2, 64
    k_pool, v_pool, k_scales, v_scales, table = [t.cuda() for t in _fp8_case(H, D, [70], seed=9)]
    qkv = torch.randn(1, H * 3 * D, device="cuda").to(torch.bfloat16)
    pos = torch.tensor([69], dtype=torch.int32, device="cuda")
    slopes = K.alibi_slopes(H, device="cuda")
    slot = torch.tensor([3], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="need k_scales"):
        alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, 69, slopes, D)
    with pytest.raises(ValueError, match="need k_scales"):
        paged_kv_write(qkv, slot, k_pool, v_pool, D)
    cu, start = torch.tensor([0, 1], dtype=torch.int32), torch.tensor([64], dtype=torch.int32)
    with pytest.raises(ValueError, match="pass stage"):              # FP8 pools are read through a staging pool
        alibi_paged_prefill_attention(qkv, k_pool, v_pool, table, cu, start, 1, slopes, D, k_scales=k_scales,
                                      v_scales=v_scales)
    bad = {"shape": k_scales[:, :, :32].contiguous(), "dtype": k_scales.half(), "device": k_scales.cpu()}
    for what, s in bad.items():
        with pytest.raises(RuntimeError):
            alibi_paged_decode_attention(qkv, k_pool, v_pool, table, pos, 69, slopes, D, k_scales=s, v_scales=v_scales)
        with pytest.raises(RuntimeError):
            paged_kv_write(qkv, slot, k_pool, v_pool, D, k_scales=s, v_scales=v_scales)
    out = torch.empty(1, H * D, device="cuda", dtype=torch.bfloat16)
    ticket = torch.zeros(64, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="bf16"):                  # FP8 pools with a non-bf16 qkv
        native().paged_decode_attention_fp8(qkv.float(), k_pool, v_pool, k_scales, v_scales, table, pos, 69, slopes,
                                            out, ticket)
    with pytest.raises(RuntimeError, match="bf16"):
        native().paged_kv_write_fp8(qkv.float(), slot, k_pool, v_pool, k_scales, v_scales)
    with pytest.raises(RuntimeError, match="bf16"):                  # the bf16 kernels refuse FP8 pools
        native().paged_decode_attention(qkv, k_pool, v_pool, table, pos, 69, slopes, out, ticket)
    with pytest.raises(RuntimeError, match="bf16"):
        native().paged_kv_write(qkv, slot, k_pool, v_pool)


# ------------------------------------------------------------------------------------------------------------ engine
def _model(arch, hidden, n_head):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    if arch == "bloom":
        model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head))
    else:
        model = GPT2LMHeadModel(GPT2Config(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head,
                                           n_positions=512))
    return model.to(torch.bfloat16).cuda().eval()


# Largest teacher-forced logit distance between FP8 and bf16 pools, over max |logit| of the step.  Measured on these
# random-init models at 0.005 - 0.012 on one H100 (e4m3 keys and values carry 3 mantissa bits: up to 2^-4 relative
# error per element, averaged down by the softmax and the projections).  The bound is about 4x that, for other seeds
# and builds; a wrong scale, a lost position or a misread page moves the logits by the order of their own size.
FP8_VS_BF16 = 0.05


@pytest.mark.parametrize("prefix_caching", [False, True])
@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_fp8_engine_against_bf16_pools_and_reference(arch, hidden, n_head, prefix_caching):
    """The FP8 engine is teacher-forced with the bf16-pool engine's tokens.  Prefills without hits: bitwise equal
    logits.  Decode steps: close to the fp32 reference path (CPU) over a copy of the same FP8 pools, and within
    FP8_VS_BF16 of the bf16-pool engine.  Shared pages are never written."""
    from pipegoose_b200.serving import ContinuousBatcher

    model = _model(arch, hidden, n_head)
    ref_model = _model(arch, hidden, n_head).float().cpu()
    g = torch.Generator().manual_seed(13)
    systems = [torch.randint(0, 4096, (n,), generator=g).tolist() for n in (130, 200)]
    prompts, news = [], []
    for i in range(10):
        n = int(torch.randint(1, 120, (1,), generator=g))
        prompts.append(systems[i % 2] + torch.randint(0, 4096, (n,), generator=g).tolist())
        news.append(int(torch.randint(2, 20, (1,), generator=g)))
    # a pool large enough that no indexed page is evicted (and rewritten) during the run
    engines = {dt: ContinuousBatcher(model, max_cache_tokens=64 * PAGE_SIZE, max_prefill_tokens=400,
                                     prefix_caching=prefix_caching, kv_cache_dtype=dt) for dt in (None, FP8)}
    logs = {dt: [] for dt in engines}
    for dt, e in engines.items():
        forward = e._forward

        def spy(forward=forward, log=logs[dt], e=e):
            kind = "prefill_hits" if e._admitted and any(r.cached for r in e._admitted) else (
                "prefill" if e._admitted else "decode")
            reqs, logits = forward()
            log.append((kind, [r.rid for r in reqs], logits.clone()))
            return reqs, logits
        e._forward = spy
    picks = {}                                             # (rid, tokens so far) -> the bf16-pool engine's pick
    select = engines[None]._select

    def lead_select(reqs, logits):
        out = select(reqs, logits)
        picks.update({(r.rid, len(r.tokens)): t for r, t in zip(reqs, out)})
        return out
    engines[None]._select = lead_select
    engines[FP8]._select = lambda reqs, logits: [picks[(r.rid, len(r.tokens))] for r in reqs]

    ref_dev = []
    paged = type(model)._paged_logits

    def checked(self, ids, positions, k_pools, v_pools, **kw):
        if kw.get("k_scales") is None or kw.get("seg_start") is not None or kw.get("start") is not None:
            return paged(self, ids, positions, k_pools, v_pools, **kw)
        snap = [t.cpu() for t in (ids, positions, k_pools, v_pools, kw["table"], kw["k_scales"], kw["v_scales"])]
        out = paged(self, ids, positions, k_pools, v_pools, **kw)
        want = paged(ref_model, snap[0], snap[1], snap[2], snap[3], table=snap[4], max_pos=kw["max_pos"],
                     k_scales=snap[5], v_scales=snap[6])
        ref_dev.append(((out.float().cpu() - want).abs().max() / want.abs().max()).item())
        return out
    model._paged_logits = checked.__get__(model)

    rids = {dt: [e.submit(p, n) for p, n in zip(prompts[:4], news[:4])] for dt, e in engines.items()}
    shared_snap = None
    for i in range(4, 10):                                 # lockstep: the bf16-pool engine's step first
        for dt, e in engines.items():
            e.step()
            rids[dt].append(e.submit(prompts[i], news[i]))
        if prefix_caching and shared_snap is None and engines[FP8]._page_key:
            shared = sorted(engines[FP8]._page_key)[:2]
            e8 = engines[FP8]
            shared_snap = (shared, [t[:, shared].clone() for t in (e8.k_pools, e8.v_pools, e8.k_scales, e8.v_scales)])
    while engines[None].has_work():
        for e in engines.values():
            e.step()
    assert not engines[FP8].has_work() and rids[None] == rids[FP8]
    del model._paged_logits

    dist = []
    assert len(logs[None]) == len(logs[FP8])
    for (kind, r16, l16), (kind8, r8, l8) in zip(logs[None], logs[FP8]):
        assert kind == kind8 and r16 == r8
        if kind == "prefill":
            assert torch.equal(l16, l8)
        else:
            dist.append(((l8 - l16).abs().max() / l16.abs().max()).item())
    print(f"\nfp8 vs bf16 pools, {arch} D={hidden // n_head} prefix_caching={prefix_caching}: max teacher-forced "
          f"logit distance {max(dist):.4f} of max |logit| over {len(dist)} steps; fp8 kernel vs fp32 reference "
          f"{max(ref_dev):.2e}")
    assert ref_dev and max(ref_dev) < 3e-2
    assert max(dist) < FP8_VS_BF16
    if prefix_caching:
        assert engines[FP8].cached_prompt_tokens > 0
        shared, before = shared_snap
        e8 = engines[FP8]
        for a, b in zip(before, (e8.k_pools, e8.v_pools, e8.k_scales, e8.v_scales)):
            assert _same(b[:, shared], a)
