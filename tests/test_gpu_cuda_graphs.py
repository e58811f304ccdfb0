"""``ContinuousBatcher(cuda_graphs=True)``: decode steps replayed from CUDA graphs.  A replay against the eager call on
the same static inputs (bitwise), capture against the live pool pages, the graph engine against the eager engine and
the training forward in every serving mode, bucket choice with the eager fallback above the largest bucket, and the
refusals (on the CPU)."""
import pytest
import torch

from pipegoose_b200 import serving
from pipegoose_b200.ops import attention as A
from pipegoose_b200.ops.attention import PAGE_SIZE
from pipegoose_b200.serving import ContinuousBatcher

FP8 = torch.float8_e4m3fn
TOL = 3e-2              # logits of two engines, and of an engine against the training forward, over max |logit|
FP8_TOL = 3e-2 + 5e-2   # FP8 pools against the training forward: TOL plus the FP8 KV-cache engine tests' bound


def _model(arch="bloom", hidden=256, n_head=4, device="cuda", dtype=torch.bfloat16):
    from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
    from pipegoose_b200.models.gpt2 import GPT2Config, GPT2LMHeadModel

    torch.manual_seed(0)
    if arch == "bloom":
        model = BloomForCausalLM(BloomConfig(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head))
    else:
        model = GPT2LMHeadModel(GPT2Config(vocab_size=4096, hidden_size=hidden, n_layer=2, n_head=n_head,
                                           n_positions=512))
    return model.to(dtype).to(device).eval()


def _workload(seed=11, n=12):
    """Requests that start with one of two shared system prompts (130 / 200 tokens), prompts up to 320 tokens and up
    to 23 new tokens: the workload of the chunked-prefill and prefix-cache engine tests."""
    g = torch.Generator().manual_seed(seed)
    systems = [torch.randint(0, 4096, (k,), generator=g).tolist() for k in (130, 200)]
    prompts, news = [], []
    for i in range(n):
        k = int(torch.randint(1, 120, (1,), generator=g))
        prompts.append(systems[i % 2] + torch.randint(0, 4096, (k,), generator=g).tolist())
        news.append(int(torch.randint(1, 24, (1,), generator=g)))
    return prompts, news


def _run(engine, prompts, news, feed=None, waves=True):
    """Submit (in waves: four, three steps, then one per step) and run to the end.  Returns the outputs by request
    index and every forward's logits ``{(rid, tokens so far): logits}``.  ``feed``: {(rid, tokens so far): token} of
    another engine's choices, taken instead of this one's where present."""
    steps = {}
    forward, select = engine._forward, engine._select

    def spy():
        reqs, logits = forward()
        for j, r in enumerate(reqs):
            steps[(r.rid, len(r.tokens))] = logits[j].clone()
        return reqs, logits
    engine._forward = spy
    if feed is not None:
        engine._select = lambda reqs, logits: [feed.get((r.rid, len(r.tokens)), t)
                                               for r, t in zip(reqs, select(reqs, logits))]
    rids, outs = {}, {}
    first = 4 if waves else len(prompts)
    for i in range(first):
        rids[i] = engine.submit(prompts[i], news[i])
    for _ in range(3 if waves else 0):
        outs.update(engine.step())
    for i in range(first, len(prompts)):
        rids[i] = engine.submit(prompts[i], news[i])
        outs.update(engine.step())
    outs.update(engine.run())
    assert len(engine._free) == engine.num_pages and engine.num_pages not in engine._free
    return {i: outs[rid] for i, rid in rids.items()}, rids, steps


def _check_against_forward(model, prompts, outs, rids, steps, tol):
    """Every recorded step's logits against the training forward on the request's final tokens, and its token against
    the arg-max wherever the top-2 margin exceeds twice the tolerance."""
    for i, rid in rids.items():
        P, out = len(prompts[i]), outs[i]
        assert P < len(out) <= P + 23
        with torch.no_grad():
            full = model(torch.tensor([out], device="cuda")).logits[0].float()
        bound = tol * full[P - 1:].abs().max().item()
        for (r, n), got in steps.items():
            if r != rid:
                continue
            want = full[n - 1]
            assert (got - want).abs().max().item() <= bound, (i, n, (got - want).abs().max().item(), bound)
            top2 = want.topk(2).values
            if n < len(out) and bool(top2[0] - top2[1] > 2 * bound):
                assert out[n] == int(want.argmax()), (i, n)


# --------------------------------------------------------------------------------------------- replay vs eager call
def _pools(engine):
    return [t for t in (engine.k_pools, engine.v_pools, engine.k_scales, engine.v_scales) if t is not None]


def _bits(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _engine_with_running(model, kv_cache_dtype, lengths=(70, 5, 200), news=(40, 40, 40)):
    """A graph engine whose requests (prompts of mixed lengths) have been prefilled and decoded for a few steps."""
    engine = ContinuousBatcher(model, max_cache_tokens=16 * PAGE_SIZE, kv_cache_dtype=kv_cache_dtype, cuda_graphs=True)
    g = torch.Generator().manual_seed(5)
    for P, N in zip(lengths, news):
        engine.submit(torch.randint(0, 4096, (P,), generator=g).tolist(), N)
    for _ in range(4):
        engine.step()
    assert len(engine._running) == len(lengths) and engine.graph_decode_steps == 3
    return engine


@pytest.mark.gpu
@pytest.mark.parametrize("kv_cache_dtype", [None, FP8])
@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_replay_is_the_eager_call(arch, hidden, n_head, kv_cache_dtype):
    """For buckets 4 and 8 with three real rows at mixed lengths: one replay and one eager ``_paged_logits`` call on the
    same static inputs (padding rows and ``max_pos`` included), from the same pools, give the same logits and leave
    the same pools, bit for bit."""
    engine = _engine_with_running(_model(arch, hidden, n_head), kv_cache_dtype)
    reqs = engine._running
    rows = ([r.tokens[-1] for r in reqs], [len(r.tokens) - 1 for r in reqs], [r.pages for r in reqs])
    assert len(set(rows[1])) == 3
    for n in (4, 8):
        graph, logits, _ = engine._graph(n)
        before = [t.clone() for t in _pools(engine)]
        engine._graph_inputs(n, *rows)
        graph.replay()
        got, got_pools = logits.clone(), [t.clone() for t in _pools(engine)]
        for t, b in zip(_pools(engine), before):
            t.copy_(b)
        want = engine._graph_call(*engine._graph_inputs(n, *rows))
        assert torch.isfinite(got).all() and torch.equal(_bits(got), _bits(want)), n
        for a, b in zip(got_pools, _pools(engine)):
            assert torch.equal(_bits(a), _bits(b)), n


@pytest.mark.gpu
@pytest.mark.parametrize("kv_cache_dtype", [None, FP8])
def test_capture_touches_no_live_page(kv_cache_dtype):
    """Capturing a new bucket while requests hold pages leaves every page but the scratch page as it was, scales
    included."""
    engine = _engine_with_running(_model(), kv_cache_dtype)
    before = [t[:, :engine.num_pages].clone() for t in _pools(engine)]
    assert 16 not in engine._graphs
    engine._graph(16)
    for t, b in zip(_pools(engine), before):
        assert torch.equal(_bits(t[:, :engine.num_pages]), _bits(b))


# --------------------------------------------------------------------------------------- graph engine vs eager engine
CONFIGS = {"plain": {}, "prefix_caching": {"prefix_caching": True},
           "chunked_prefill": {"chunked_prefill": True, "max_prefill_tokens": 128},
           "fp8": {"kv_cache_dtype": FP8}, "speculative": {"num_speculative_tokens": 4}}


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("arch,hidden,n_head", [("bloom", 256, 4), ("bloom", 320, 4), ("bloom", 512, 4),
                                                  ("gpt2", 256, 4)])
def test_graph_engine_matches_eager_engine(arch, hidden, n_head, config):
    """The graph engine, fed the eager engine's tokens, gives every decode step's logits within TOL of the eager
    engine's, and both agree with the training forward."""
    model = _model(arch, hidden, n_head)
    prompts, news = _workload()
    kw = dict(CONFIGS[config], max_cache_tokens=24 * PAGE_SIZE)
    eager = ContinuousBatcher(model, **kw)
    graphs = ContinuousBatcher(model, cuda_graphs=True, **kw)
    outs_e, rids_e, steps_e = _run(eager, prompts, news)
    feed = {(rids_e[i], n): out[n] for i, out in outs_e.items() for n in range(len(prompts[i]), len(out))}
    outs_g, rids_g, steps_g = _run(graphs, prompts, news, feed=feed)
    assert rids_g == rids_e and eager.graph_decode_steps == 0 and graphs.graph_decode_steps > 0
    if config != "speculative":              # verify steps accept drafts by their own arg-max
        assert outs_g == outs_e
    common = set(steps_e) & set(steps_g)
    assert len(common) > len(prompts)
    for key in common:
        e, g = steps_e[key], steps_g[key]
        assert (g - e).abs().max().item() <= TOL * e.abs().max().item(), (key, (g - e).abs().max().item())
    tol = FP8_TOL if config == "fp8" else TOL
    _check_against_forward(model, prompts, outs_e, rids_e, steps_e, tol)
    _check_against_forward(model, prompts, outs_g, rids_g, steps_g, tol)


# ------------------------------------------------------------------------------------------- buckets and fallback
@pytest.mark.gpu
def test_buckets_and_eager_fallback(monkeypatch):
    """Buckets (1, 2, 4): four requests decode by replay of bucket 4, five decode eagerly once bucket 4 is captured
    (their step needs more decode tickets than the exactly-sized array bucket 4 was captured with, so the cached array
    is replaced), and three replay bucket 4 again, with the array it captured.  Results match the eager engine and the
    training forward; the free list ends full and never holds the scratch page."""
    monkeypatch.setattr(serving, "GRAPH_BATCH_SIZES", (1, 2, 4))
    model = _model()
    H = model.config.n_head
    prompts, news = _workload(seed=3, n=5)
    news = [20, 8, 14, 20, 16]                   # 5 running, then 3 after two finish
    eager = ContinuousBatcher(model, max_cache_tokens=40 * PAGE_SIZE)
    outs_e, rids_e, steps_e = _run(eager, prompts, news, waves=False)

    device = next(model.parameters()).device
    seeded = torch.zeros(4 * H, dtype=torch.int32, device=device)
    monkeypatch.setitem(A._decode_tickets, device, seeded)
    engine = ContinuousBatcher(model, max_cache_tokens=40 * PAGE_SIZE, cuda_graphs=True)
    steps_g, sizes, replayed = {}, [], []
    forward, graph_decode = engine._forward, engine._graph_decode

    def spy_forward():
        decode = not engine._admitted
        reqs, logits = forward()
        if decode and reqs:
            sizes.append(len(reqs))
        for j, r in enumerate(reqs):
            steps_g[(r.rid, len(r.tokens))] = logits[j].clone()
        return reqs, logits

    def spy_graph(reqs):
        replayed.append(len(reqs))
        return graph_decode(reqs)
    feed = {(rids_e[i], n): out[n] for i, out in outs_e.items() for n in range(len(prompts[i]), len(out))}
    engine._forward, engine._graph_decode = spy_forward, spy_graph
    engine._select = lambda reqs, logits: [feed[(r.rid, len(r.tokens))] for r in reqs]

    rids = {i: engine.submit(prompts[i], news[i]) for i in range(4)}
    outs = dict(engine.step())                    # prefill
    outs.update(engine.step())                    # bucket 4 captured with the seeded ticket array
    assert engine._graphs[4][2] is seeded and replayed == [4]
    rids[4] = engine.submit(prompts[4], news[4])
    outs.update(engine.run())
    assert 5 in sizes and 5 not in replayed and 3 in replayed
    assert A._decode_tickets[device] is not seeded and engine._graphs[4][2] is seeded
    assert rids == rids_e and {i: outs[rid] for i, rid in rids.items()} == outs_e
    assert len(engine._free) == engine.num_pages and engine.num_pages not in engine._free
    assert engine.graph_decode_steps == len(replayed)
    assert set(steps_g) == set(steps_e)
    for key, e in steps_e.items():
        assert (steps_g[key] - e).abs().max().item() <= TOL * e.abs().max().item(), key
    _check_against_forward(model, prompts, outs_e, rids, steps_g, TOL)


# ------------------------------------------------------------------------------------------------------- refusals
def test_refusals_on_the_cpu():
    """Models off the native decode path, and models with ExpertLayer MLPs, are refused at construction; without the
    option the pools keep ``num_pages`` pages."""
    from pipegoose_b200.nn.expert_parallel.layers import ExpertLayer

    for dtype in (torch.bfloat16, torch.float32):
        with pytest.raises(ValueError, match="native decode path"):
            ContinuousBatcher(_model(device="cpu", dtype=dtype), max_cache_tokens=PAGE_SIZE, cuda_graphs=True)
    moe = _model(device="cpu", dtype=torch.float32)
    moe.transformer.h[1].mlp = ExpertLayer(2, torch.nn.Linear(256, 256), None, True, None)
    with pytest.raises(ValueError, match="ExpertLayer"):
        ContinuousBatcher(moe, max_cache_tokens=PAGE_SIZE, cuda_graphs=True)
    engine = ContinuousBatcher(moe, max_cache_tokens=3 * PAGE_SIZE)
    assert engine.k_pools.shape[1] == engine.num_pages == 3 and engine.graph_decode_steps == 0


@pytest.mark.gpu
def test_refusals_on_the_gpu():
    for model in (_model(dtype=torch.float32), _model(hidden=128, n_head=4)):       # fp32; head size 32
        with pytest.raises(ValueError, match="native decode path"):
            ContinuousBatcher(model, max_cache_tokens=PAGE_SIZE, cuda_graphs=True)
