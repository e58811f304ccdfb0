"""The attention kernels against one float64 reference, element by element, on inputs where every key counts.

Every kernel computes the same thing: query i of head h sits at position p_i and sees keys lo_i <= k <= hi_i (hi_i =
p_i) with the score ``q.k * scale + slope_h * (k - p_i)``.  :func:`attend` computes that in float64 from the values the
kernel reads; thin adapters turn each layout (the flash kernels' fused ``[B*S, H*3*D]`` rows with ``seg_start``, the
contiguous decode cache with ``lead``, the paged pools with their table, ``pos`` / ``cu_seqlens`` / ``start``) into
that form.  Over FP8 pools the reference reads exactly what the kernel reads: ``float(code) * scale`` in the decode
kernel, ``bf16(float(code) * scale)`` in the prefill kernel's staging pool (``kv_dequantize_kernel``), and the step's
own tokens exactly, from ``qkv``.  Quantization is an input to the reference, not part of the bound.  The backward
reference is float64 autograd through :func:`attend`.  The references run on the device in the GPU tests.

Bounds
------
Each check is ``|got - want| <= atol + 2^-8 |want|`` (``2^-8``: the bf16 output rounding; ``lse`` is fp32 and has
rtol 0).  ``u = 2^-24``; p_ik are the exact probabilities, A_id = sum_k p_ik |v_kd|, and scores are in log2 units
(x = score * log2e) as the kernels compute them.

* Score error dx_ik.  The fp32 dot product over D carries ``n_dot * u * scale * log2e * sum_d |q_d k_d|``, with n_dot
  the chain depth plus the roundings of ``scale_log2`` (log2e, 1/sqrtf(D), their product) and of the pre-scaled q: in
  the decode kernels 8 sequential fmas (16 over FP8 codes, +1 for ``dot * s_k``) and log2(lanes per key) shuffle adds;
  in the tensor-core kernels D (wgmma's internal order is not documented, so the sequential bound over all D).  The
  ALiBi term ``slope * log2e * (k - p)`` carries 2u (decode: slope_log2, fma) or 3u (flash: slope2, ``bias0`` formed at
  the block's first key -- hence the distance padded by a block, 128 -- and the fma) of ``|slope log2e| (|k - p| + pad)``.
  The subtraction of the running maximum and the rescales of earlier keys carry at most 2u (M - x_k).  A score error
  moves out_id by at most ``ln2 * sum_k p_ik dx_ik |v_kd - out_id|``; the bound uses |v - o| <= |v| + |o|, which keeps it
  two matrix products.
* exp2 error.  ``exp2f`` (decode family) and ``ex2.approx.ftz.f32`` (``fast_exp2``, flash family) are both documented
  at 2 ulp, a relative 2^-22.  Every p carries one, and so does every rescale applied to it afterwards (one per key
  iteration, NG * kDecUnroll keys, in the decode kernels; one per 128-key block in the flash kernels) plus the merges
  of key groups and splits.  A relative error e on the weights moves out by e (A + |o|).
* Underflow.  A weight below 2^-126 of the row maximum is flushed (``ftz``) or kept as an fp32 denormal, and every
  product and sum near that range loses its relative precision: an absolute ``(n + 4) 2^-126 max |v|`` per output,
  with n visible keys.  It matters only where the exact output is itself that small, as in regime F's columns fed
  only by far chunks of the steep heads.
* Accumulation.  Decode family (everything in fp32 registers): per key group ceil(n / NG) fmas into o and l plus one
  rescale multiply per iteration, a merge over NG groups and one over at most ceil(n / 64) splits (kDecMinChunk = 64,
  so the bound does not depend on the split plan), and the division: depth * u * (A + |o|).  Tensor-core family: the
  fp32 accumulator over all n visible keys plus a rescale per block: (n + blocks + 8) u (A + |o|); P is rounded to
  bf16 before P.V while l sums the unrounded p, which adds 2^-8 A_id.  (The rounding of p in [2^e, 2^(e+1)) to 8
  significant bits moves it by up to 2^-8 of itself: 2^-9 would be the rounding of a value at the bottom of its binade
  only, so the bound takes the unit roundoff of bf16.)
* ``lse`` (flash forward, natural log): ``ln2 * sum_k p_k dx_k`` (the first-order change of logsumexp), the exp2 and
  accumulation terms of l, 2^-22 log2(n) for ``log2f``, and 3u |lse| for the add and the multiply by ln2.
* Backward.  The kernel recomputes p = exp2(x - lse * log2e) with its own score error (the forward's, plus 2u
  (|x| + |lse2|) for the fmas that fold in -lse2) and the forward's lse error, a relative rho_ij.  dV_j = sum_i p_ij dO_i
  gets ``sum_i p_ij (rho_ij + 2^-8) |dO_i|`` (the bf16 P^T) plus accumulation.  dS = p (dP - delta) scale, where dP's
  D-long dot product carries (D + 6) u sum_d |dO_d V_jd| and delta is computed from the bf16 ``out``:
  ``sum_d |dO_id| (atol_out_id + 2^-8 |O_id|)``.  dS is rounded to bf16 (2^-8 |dS|) before dK = dS^T Q and dQ = dS K,
  which get sum |delta dS| |q| (or |k|) plus (S + 4) u sum |dS| |q| (or |k|).  The bf16 output rounding is the rtol.

Set ``PIPEGOOSE_ERROR_REPORT=<path>`` to write the largest ``|err| / bound`` of every check to JSON.

Regimes
-------
* R: ``alibi_slopes`` and randn: the realistic case, where the steep heads set the scale and far keys weigh little.
* F (flat): slopes 0 on the even heads (the odd ones keep ALiBi), q = 0.25 randn so attention spreads over every
  visible key, and ``V[k, d] = 1 if (k // 64) % D == d else 0``: each output column is the attention mass of its own
  64-key chunks, so a dropped, duplicated or misplaced chunk, page, split or 128-key block moves some column by a large
  fraction of itself.
* N (needles): slopes 0, random K, and q_i = c k_t(i) in bf16 with c chosen so that the target leads every other key
  of the row by about 20 nats.  The targets alternate between a key just outside the visible range (p_i + 1,
  ``seg_start - 1``, the next document's first key; for decode rows an unused slot, which holds a decoy in one run) --
  a leak moves the output to v_t -- and the first visible key of the range or of a chunk half way back -- dropping it
  changes the output by O(1).

The ``test_bounds_reject_*`` tests apply plausible kernel mistakes to the float64 reference on each regime's inputs and
require the bound to be exceeded at least 10 times over in some element, in the regime meant to catch each mistake.
A 64-key chunk is no larger than any split (kDecMinChunk), page or flash block, so these emulations do not depend on
the split plan.
"""
import json
import math
import os

import pytest
import torch

from pipegoose_b200.ops import kernels as K
from pipegoose_b200.ops.attention import (
    PAGE_SIZE, alibi_attention, alibi_attention_reference, alibi_decode_attention, alibi_decode_attention_reference,
    alibi_paged_append_attention, alibi_paged_append_attention_reference, alibi_paged_decode_attention,
    alibi_paged_decode_attention_reference, alibi_paged_prefill_attention, fp8_prefill_staging, pad_heads,
    padded_head_dim, paged_prefill_attention_fp32, quantize_kv, unpad_heads)

gpu = pytest.mark.gpu

U32 = 2.0 ** -24      # fp32 unit roundoff
UBF = 2.0 ** -8       # bf16 unit roundoff
EXP_ERR = 2.0 ** -22  # exp2f and ex2.approx.ftz.f32: 2 ulp
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
TINY = 2.0 ** -126    # smallest normal fp32
MARGIN = 10.0         # a mistake must exceed its bound at least this many times over
FP8 = torch.float8_e4m3fn
REGIMES = ["R", "F", "N"]
DEC_LENGTHS = [1, 2, 63, 64, 65, 1000, 4097, 33000]
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
    """Largest ``|got - want| / (atol + rtol |want|)``; inf where ``got`` is not finite and ``want`` is."""
    got, want = got.double(), want.double().to(got.device)
    atol = torch.as_tensor(atol, dtype=torch.float64, device=got.device)
    err = (got - want).abs()
    err = torch.where(got == want, torch.zeros_like(err), err)
    err = torch.where(torch.isfinite(got) | ~torch.isfinite(want), err, torch.full_like(err, math.inf))
    r = torch.where(err == 0, torch.zeros_like(err), err / (atol + rtol * want.abs()))
    return r.max().item() if r.numel() else 0.0


def _check(name, got, want, atol, rtol=UBF):
    r = _ratio(got, want, atol, rtol)
    _WORST[name] = max(_WORST.get(name, 0.0), r)
    assert r <= 1.0, f"{name}: largest |err| / bound is {r:.3g}"


def _bf(x):
    """float64 values of bf16 roundings."""
    return x.to(torch.bfloat16).double()


# ================================================================================================================
# float64 reference and bounds
# ================================================================================================================
def attend(q, k, v, lo, hi, slopes, scale, qpos=None, logw=None):
    """Queries ``q [H, n, D]`` over keys ``k`` / ``v [H, m, D]`` at positions 0 .. m-1, in float64: query i sees keys
    ``lo[i] <= j <= hi[i]`` with the score ``q.k * scale + slope[h] * (j - qpos[i])`` (``qpos`` defaults to ``hi``);
    ``logw`` (broadcast to ``[H, n, m]``) is added to the scores.  Returns ``out [H, n, D]``, ``lse [H, n]`` (natural
    log) and the probabilities ``p [H, n, m]``."""
    m = k.shape[1]
    qpos = hi if qpos is None else qpos
    j = torch.arange(m, device=k.device)
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    s = s + slopes.double().to(k.device).view(-1, 1, 1) * (j.view(1, 1, -1) - qpos.view(1, -1, 1)).double()
    if logw is not None:
        s = s + logw
    vis = (j.view(1, -1) >= lo.view(-1, 1)) & (j.view(1, -1) <= hi.view(-1, 1))
    s = s.masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse.unsqueeze(-1))
    return torch.matmul(p, v), lse, p


class Family:
    """Arithmetic of a kernel family (module docstring): ``n_dot`` roundings on the dot product, ``n_slope`` on the
    ALiBi term with its distance padded by ``pad``, per-key exp2 and accumulation depths for ``n`` visible keys, and
    whether P is rounded to bf16 before P.V."""

    def __init__(self, n_dot, n_slope, pad, exp_depth, acc_depth, p_bf16):
        self.n_dot, self.n_slope, self.pad = n_dot, n_slope, pad
        self.exp_depth, self.acc_depth, self.p_bf16 = exp_depth, acc_depth, p_bf16


def decode_family(D, fp8=False, unroll=4):
    lanes = D // 16 if fp8 else D // 8
    lpk = (4 if lanes <= 4 else 8) if fp8 else (8 if lanes <= 8 else 16)
    ng = 4 * (32 // lpk)
    n_dot = (17 if fp8 else 8) + int(math.log2(lpk)) + 6
    iters = lambda n: -(-n // (ng * unroll))
    return Family(n_dot, 2, 0, lambda n: 4 + iters(n),
                  lambda n: -(-n // ng) + iters(n) + ng + -(-n // 64) + 4 + fp8, False)


def flash_family(D):
    blocks = lambda n: -(-n // 128) + 1
    return Family(D + 6, 3, 128, lambda n: 2 + blocks(n), lambda n: n + blocks(n) + 8, True)


def fwd_bounds(q, k, v, lo, hi, slopes, scale, out, lse, p, fam, qpos=None):
    """``atol`` of ``out [H, n, D]`` and of ``lse [H, n]`` for the kernel family ``fam`` (module docstring)."""
    m = k.shape[1]
    qpos = hi if qpos is None else qpos
    j = torch.arange(m, device=k.device)
    dist = (j.view(1, -1) - qpos.view(-1, 1)).abs().double() + fam.pad
    qk = torch.matmul(q.abs(), k.abs().transpose(-1, -2)) * (scale * LOG2E)
    gap = torch.where(p > 0, -torch.log(p.clamp_min(1e-300)) * LOG2E, torch.zeros_like(p))   # >= M - x_k
    dx = (fam.n_dot * U32) * qk + (fam.n_slope * U32) * slopes.double().abs().to(k.device).view(-1, 1, 1) * LOG2E \
        * dist + (2 * U32) * gap
    pdx = p * dx * LN2
    A = torch.matmul(p, v.abs())
    score = torch.matmul(pdx, v.abs()) + out.abs() * pdx.sum(-1, keepdim=True)
    n = (hi - lo + 1).tolist()
    rel = torch.tensor([fam.exp_depth(x) * EXP_ERR + fam.acc_depth(x) * U32 for x in n], dtype=torch.float64,
                       device=k.device).view(1, -1)
    vmax = v.abs().amax(dim=(0, 1, 2)).item() if v.numel() else 0.0
    floor = torch.tensor([(x + 4) * TINY * vmax for x in n], dtype=torch.float64, device=k.device).view(1, -1, 1)
    atol = score + rel.unsqueeze(-1) * (A + out.abs()) + (UBF * A if fam.p_bf16 else 0.0) + floor
    logn = torch.tensor([math.log2(max(x, 1)) for x in n], dtype=torch.float64, device=k.device).view(1, -1)
    atol_lse = pdx.sum(-1) + rel + EXP_ERR * logn + 3 * U32 * lse.abs()
    return atol, atol_lse


# ================================================================================================================
# Regimes
# ================================================================================================================
def regime_slopes(regime, H):
    s = K.alibi_slopes(H)
    if regime == "N":
        return torch.zeros(H)
    if regime == "F":
        s[0::2] = 0.0
    return s


def needle_target(i, lo, hi, m):
    """The key query number ``i`` points at in regime N: alternately just outside its range (after it, then before
    it) and the first visible key of its range or of a chunk half way back."""
    kind = i % 4
    if kind in (0, 2):
        out = [hi + 1, lo - 1] if kind == 0 else [lo - 1, hi + 1]
        for t in out:
            if 0 <= t < m and not lo <= t <= hi:
                return t
    if kind == 1 or hi - lo < 128:
        return lo
    return lo + 64 * ((hi - lo) // 128)


def gen_seq(regime, H, D, m, lo, hi, g, scale, first=0):
    """One sequence of ``m`` keys and the queries at ranges ``[lo[i], hi[i]]``: float64 bf16-valued ``q [H, n, D]``,
    ``k``, ``v [H, m, D]``.  ``first`` numbers the queries for the alternation of needle kinds."""
    n = len(hi)
    k = _bf(torch.randn(H, m, D, generator=g, dtype=torch.float64))
    if regime == "F":
        v = torch.zeros(H, m, D, dtype=torch.float64)
        v[:, torch.arange(m), (torch.arange(m) // 64) % D] = 1.0
    else:
        v = _bf(torch.randn(H, m, D, generator=g, dtype=torch.float64))
    if regime == "N":
        q = torch.empty(H, n, D, dtype=torch.float64)
        for i in range(n):
            t = needle_target(first + i, int(lo[i]), int(hi[i]), m)
            kt = k[:, t]                                                     # [H, D]
            dots = torch.einsum("hd,hmd->hm", kt, k)
            dots[:, t] = -math.inf
            gap = (kt * kt).sum(-1) - dots.max(-1).values                   # > 0 for random keys
            q[:, i] = _bf(kt * (20.0 / (scale * gap)).view(H, 1))
    else:
        q = _bf(torch.randn(H, n, D, generator=g, dtype=torch.float64) * (0.25 if regime == "F" else 1.0))
    return q, k, v


def decoy_rows(q):
    """Decoy keys / values for unused slots: keys along the row's query, about 24 nats above zero, values 4."""
    c = 24.0 / (q * q).sum(-1, keepdim=True).clamp_min(1e-3)
    return _bf(q * c), torch.full_like(q, 4.0)


# ================================================================================================================
# CPU: the reference against independent computations, and the fp32 references of ops/attention.py against it
# ================================================================================================================
def test_reference_matches_explicit_softmax_and_sdpa():
    g = torch.Generator().manual_seed(0)
    H, m, D = 3, 70, 16
    q, k, v = (torch.randn(H, m, D, generator=g, dtype=torch.float64) for _ in range(3))
    slopes = torch.tensor([0.0, 0.25, 2.0 ** -8], dtype=torch.float64)
    lo = torch.tensor([max(0, i - 5 * (i % 7)) for i in range(m)])
    hi = torch.arange(m)
    out, lse, p = attend(q, k, v, lo, hi, slopes, 0.3)
    for h in range(H):
        for i in range(m):
            js = range(int(lo[i]), i + 1)
            s = [float(q[h, i] @ k[h, j]) * 0.3 + float(slopes[h]) * (j - i) for j in js]
            mx = max(s)
            w = [math.exp(x - mx) for x in s]
            l = sum(w)
            want = sum(wj * v[h, j] for wj, j in zip(w, js)) / l
            assert torch.allclose(out[h, i], want, rtol=1e-13, atol=1e-13)
            assert abs(float(lse[h, i]) - (mx + math.log(l))) < 1e-12
    j = torch.arange(m)
    bias = slopes.view(H, 1, 1) * (j.view(1, 1, -1) - hi.view(1, -1, 1)).double()
    bias = bias.masked_fill((j.view(1, -1) < lo.view(-1, 1)) | (j.view(1, -1) > hi.view(-1, 1)), -math.inf)
    sdpa = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=bias, scale=0.3)
    assert torch.allclose(out, sdpa, rtol=1e-12, atol=1e-12)


FP32_REF = Family(40, 3, 0, lambda n: 4, lambda n: n + 8, False)   # torch's fp32 matmul / softmax, loosely


def _check_fp32(name, got, want, atol):
    """An fp32 reference against the float64 one: the fp32 arithmetic bound plus fp32 output rounding."""
    _check(name, got, want, atol + 1e-30, U32)


@pytest.mark.parametrize("regime", REGIMES)
def test_fp32_flash_reference(regime):
    g = torch.Generator().manual_seed(1)
    B, S, H, D = 2, 150, 2, 32
    scale = 1 / math.sqrt(D)
    seg = torch.tensor([[0] * 40 + [40] * 110, [0] * 63 + [63] + [64] * 86], dtype=torch.int32)
    slopes = regime_slopes(regime, H)
    rows = []
    for b in range(B):
        q, k, v = gen_seq(regime, H, D, S, seg[b].long(), torch.arange(S), g, scale)
        rows.append(torch.stack([q, k, v], 2).transpose(0, 1))              # [S, H, 3, D]
    qkv = torch.stack(rows).reshape(B * S, H * 3 * D)
    got = alibi_attention_reference(qkv.float(), slopes, B, S, H, D, seg_start=seg).view(B, S, H, D)
    for b in range(B):
        x = qkv.view(B, S, H, 3, D)[b].transpose(0, 1)
        args = (x[:, :, 0], x[:, :, 1], x[:, :, 2], seg[b].long(), torch.arange(S), slopes, scale)
        out, lse, p = attend(*args)
        atol, _ = fwd_bounds(*args, out, lse, p, FP32_REF)
        _check_fp32(f"fp32_ref/flash/{regime}", got[b].transpose(0, 1), out, atol)


def _decode_layout(regime, H, D, cap, pos, leads, g, scale):
    """Contiguous caches ``[B, H, cap, D]`` holding every row's keys at every slot, the step's qkv rows and the
    float64 per-row (q, k, v)."""
    B = len(leads)
    seqs = [gen_seq(regime, H, D, cap, torch.tensor([min(l, pos)]), torch.tensor([pos]), g, scale, first=b)
            for b, l in enumerate(leads)]
    kc = torch.stack([s[1] for s in seqs])
    vc = torch.stack([s[2] for s in seqs])
    qkv = torch.stack([torch.stack([s[0][:, 0], s[1][:, pos], s[2][:, pos]], 1) for s in seqs]).view(B, H * 3 * D)
    return qkv, kc, vc, seqs


@pytest.mark.parametrize("regime", REGIMES)
def test_fp32_decode_reference(regime):
    g = torch.Generator().manual_seed(2)
    H, D, cap, pos = 2, 32, 300, 260
    scale = 1 / math.sqrt(D)
    leads = [0, 7, 400]
    slopes = regime_slopes(regime, H)
    qkv, kc, vc, seqs = _decode_layout(regime, H, D, cap, pos, leads, g, scale)
    got = alibi_decode_attention_reference(qkv.float(), kc.float(), vc.float(), slopes, pos,
                                           torch.tensor(leads), D).view(3, H, D)
    for b, (q, k, v) in enumerate(seqs):
        args = (q, k, v, torch.tensor([min(leads[b], pos)]), torch.tensor([pos]), slopes, scale)
        out, lse, p = attend(*args)
        atol, _ = fwd_bounds(*args, out, lse, p, FP32_REF)
        _check_fp32(f"fp32_ref/decode/{regime}", got[b].unsqueeze(1), out, atol)


def build_pools(seqs, lengths, H, D, fill, g, spare=3, fp8=False, dev="cpu", stored=None):
    """Paged pools over a shuffled page table with pages for positions ``0 .. lengths[r] - 1`` of every sequence, holding
    sequence r's keys / values ``seqs[r] = (q, k, v)`` at positions ``0 .. stored[r] - 1`` (default: all).  Every other slot holds ``fill``: "nan", or "decoy" (:func:`decoy_rows` of the row's first
    query; spare pages take row 0's).  FP8 pools hold ``quantize_kv`` codes and scales.  Returns the pools (and scales),
    the table and the float64 keys / values the kernels read from them (dequantized for FP8 as ``float(code) * scale``)."""
    stored = lengths if stored is None else stored
    need = [max(1, -(-n // PAGE_SIZE)) for n in lengths]
    num = sum(need) + spare
    perm = torch.randperm(num, generator=g)
    table = torch.full((len(lengths), max(need) + 1), -7, dtype=torch.int32)
    kf = torch.full((num, H, PAGE_SIZE, D), math.nan, dtype=torch.float64)
    vf = kf.clone()
    if fill == "decoy":
        dk, dv = decoy_rows(seqs[0][0][:, 0])
        kf[:], vf[:] = dk.view(1, H, 1, D), dv.view(1, H, 1, D)
    used = 0
    for r, ((q, k, v), n) in enumerate(zip(seqs, stored)):
        pages = perm[used:used + need[r]]
        table[r, :need[r]] = pages.to(torch.int32)
        used += need[r]
        if fill == "decoy":
            dk, dv = decoy_rows(q[:, 0])
            kf[pages], vf[pages] = dk.view(1, H, 1, D), dv.view(1, H, 1, D)
        p = torch.arange(n)
        kf[pages[p // PAGE_SIZE], :, p % PAGE_SIZE] = k[:, :n].transpose(0, 1)
        vf[pages[p // PAGE_SIZE], :, p % PAGE_SIZE] = v[:, :n].transpose(0, 1)
    if not fp8:
        return (kf.to(torch.bfloat16).to(dev), vf.to(torch.bfloat16).to(dev)), table.to(dev), kf, vf
    (kc, ks), (vc, vs) = quantize_kv(kf.float()), quantize_kv(vf.float())     # NaN rows: codes 0, scale NaN
    deq = lambda c, s: c.double() * s.double().unsqueeze(-1)
    return (kc.to(dev), vc.to(dev), ks.to(dev), vs.to(dev)), table.to(dev), deq(kc, ks), deq(vc, vs)


def paged_rows(pool64, table_row, n):
    """float64 ``[H, n, D]`` rows of positions ``0 .. n-1`` read through one table row."""
    p = torch.arange(n, device=pool64.device)
    return pool64[table_row.long().to(pool64.device)[p // PAGE_SIZE], :, p % PAGE_SIZE].transpose(0, 1)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("regime", REGIMES)
def test_fp32_paged_decode_reference(regime, fp8):
    g = torch.Generator().manual_seed(3)
    H, D = 2, 32
    scale = 1 / math.sqrt(D)
    lengths = [1, 65, 200]
    slopes = regime_slopes(regime, H)
    seqs = [gen_seq(regime, H, D, n, torch.tensor([0]), torch.tensor([n - 1]), g, scale, first=b)
            for b, n in enumerate(lengths)]
    pools, table, kf, vf = build_pools(seqs, lengths, H, D, "decoy", g, fp8=fp8, stored=[n - 1 for n in lengths])
    qkv = torch.stack([torch.stack([q[:, 0], k[:, -1], v[:, -1]], 1) for q, k, v in seqs]).view(3, H * 3 * D)
    pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32)
    kw = dict(k_scales=pools[2], v_scales=pools[3]) if fp8 else {}
    got = alibi_paged_decode_attention_reference(qkv.float(), pools[0] if fp8 else pools[0].float(),
                                                 pools[1] if fp8 else pools[1].float(), table, pos, 199, slopes, D,
                                                 **kw).view(3, H, D)
    for b, ((q, k, v), n) in enumerate(zip(seqs, lengths)):
        kk, vv = paged_rows(kf, table[b], n), paged_rows(vf, table[b], n)
        kk[:, n - 1], vv[:, n - 1] = k[:, n - 1], v[:, n - 1]               # the step's own token, exact
        args = (q, kk, vv, torch.tensor([0]), torch.tensor([n - 1]), slopes, scale)
        out, lse, p = attend(*args)
        atol, _ = fwd_bounds(*args, out, lse, p, FP32_REF)
        _check_fp32(f"fp32_ref/paged_decode/{regime}/fp8={fp8}", got[b].unsqueeze(1), out, atol)


def _prefill_layout(regime, H, D, starts, news, fill, g, scale, fp8=False, dev="cpu", bf16_tiles=True):
    """Pools holding every sequence's positions before ``start`` (and, over bf16 pools, its new tokens too), the new
    tokens' packed qkv, and per sequence the float64 (q, k, v) the kernels read: over FP8 pools the cached positions
    as ``bf16(float(code) * scale)`` (``bf16_tiles``; otherwise ``float(code) * scale``) and the new ones exactly."""
    seqs, first = [], 0
    for s, n in zip(starts, news):
        seqs.append(gen_seq(regime, H, D, s + n, torch.zeros(n, dtype=torch.long), torch.arange(s, s + n), g, scale,
                            first=first))
        first += n
    lengths = [s + n for s, n in zip(starts, news)]
    pools, table, kf, vf = build_pools(seqs, lengths, H, D, fill, g, fp8=fp8, dev=dev,
                                       stored=starts if fp8 else lengths)
    if fp8 and bf16_tiles:       # kv_dequantize_kernel: the fp32 product, rounded to bf16
        kf, vf = ((c.float().cpu() * s.cpu().unsqueeze(-1)).to(torch.bfloat16).double() for c, s in
                  ((pools[0], pools[2]), (pools[1], pools[3])))
    qkv = torch.cat([torch.stack([q, k[:, s:], v[:, s:]], 2).transpose(0, 1).reshape(n, H * 3 * D)
                     for (q, k, v), s, n in zip(seqs, starts, news)])
    refs = []
    for r, ((q, k, v), s, n) in enumerate(zip(seqs, starts, news)):
        kk, vv = paged_rows(kf, table[r].cpu(), s + n), paged_rows(vf, table[r].cpu(), s + n)
        if fp8:
            kk[:, s:], vv[:, s:] = k[:, s:], v[:, s:]
        refs.append((q, kk, vv, torch.zeros(n, dtype=torch.long), torch.arange(s, s + n)))
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32)
    return qkv, pools, table, cu, torch.tensor(starts, dtype=torch.int32), refs


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("regime", REGIMES)
def test_fp32_paged_prefill_reference(regime, fp8):
    g = torch.Generator().manual_seed(4)
    H, D = 2, 32
    scale = 1 / math.sqrt(D)
    starts, news = [0, 64, 128], [3, 70, 1]
    slopes = regime_slopes(regime, H)
    qkv, pools, table, cu, st, refs = _prefill_layout(regime, H, D, starts, news, "nan", g, scale, fp8=fp8,
                                                      bf16_tiles=False)
    kw = dict(k_scales=pools[2], v_scales=pools[3]) if fp8 else {}
    kp, vp = (pools[0], pools[1]) if fp8 else (pools[0].float(), pools[1].float())
    got = paged_prefill_attention_fp32(qkv.float(), kp, vp, table, cu, st, 70, slopes, D, **kw).view(-1, H, D)
    for r, ref in enumerate(refs):
        out, lse, p = attend(*ref, slopes, scale)
        atol, _ = fwd_bounds(*ref, slopes, scale, out, lse, p, FP32_REF)
        _check_fp32(f"fp32_ref/paged_prefill/{regime}", got[int(cu[r]):int(cu[r + 1])].transpose(0, 1), out, atol)


@pytest.mark.parametrize("regime", REGIMES)
def test_fp32_append_reference(regime):
    g = torch.Generator().manual_seed(5)
    H, D = 2, 32
    scale = 1 / math.sqrt(D)
    starts, news = [0, 63, 130], [2, 8, 1]
    slopes = regime_slopes(regime, H)
    qkv, pools, table, cu, st, refs = _append_layout(regime, H, D, starts, news, "nan", g, scale)
    got = alibi_paged_append_attention_reference(qkv.float(), pools[0].float(), pools[1].float(), table, cu, st, 140,
                                                 slopes, D).view(-1, H, D)
    for r, ref in enumerate(refs):
        out, lse, p = attend(*ref, slopes, scale)
        atol, _ = fwd_bounds(*ref, slopes, scale, out, lse, p, FP32_REF)
        _check_fp32(f"fp32_ref/append/{regime}", got[int(cu[r]):int(cu[r + 1])].transpose(0, 1), out, atol)


def _append_layout(regime, H, D, starts, news, fill, g, scale, dev="cpu"):
    """As :func:`_prefill_layout` over bf16 pools that hold the cached positions only (the append op writes the new
    tokens itself)."""
    seqs, first = [], 0
    for s, n in zip(starts, news):
        seqs.append(gen_seq(regime, H, D, s + n, torch.zeros(n, dtype=torch.long), torch.arange(s, s + n), g, scale,
                            first=first))
        first += n
    pools, table, kf, vf = build_pools(seqs, [s + n for s, n in zip(starts, news)], H, D, fill, g, dev=dev,
                                       stored=starts)
    qkv = torch.cat([torch.stack([q, k[:, s:], v[:, s:]], 2).transpose(0, 1).reshape(n, H * 3 * D)
                     for (q, k, v), s, n in zip(seqs, starts, news)])
    refs = [(q, k, v, torch.zeros(n, dtype=torch.long), torch.arange(s, s + n))
            for (q, k, v), s, n in zip(seqs, starts, news)]
    cu = torch.tensor([0] + torch.tensor(news).cumsum(0).tolist(), dtype=torch.int32)
    return qkv, pools, table, cu, torch.tensor(starts, dtype=torch.int32), refs


# ================================================================================================================
# CPU: the bounds reject plausible kernel mistakes (float64 emulations on each regime's inputs)
# ================================================================================================================
def _worst_ratio(bad, want, atol):
    return _ratio(bad, want, atol, UBF)


def _chunk_logw(m, c, value):
    w = torch.zeros(m, dtype=torch.float64)
    w[64 * c:64 * c + 64] = value
    return w


def _decode_case(regime, L, D=64, H=4, lead=0, first=1, seed=11):
    g = torch.Generator().manual_seed(seed + L)
    scale = 1 / math.sqrt(D)
    q, k, v = gen_seq(regime, H, D, L + 1, torch.tensor([lead]), torch.tensor([L - 1]), g, scale, first=first)
    return (q, k, v, torch.tensor([lead]), torch.tensor([L - 1]), regime_slopes(regime, H), scale)


def _flash_case(regime, S=300, D=64, H=4, seed=12):
    g = torch.Generator().manual_seed(seed)
    scale = 1 / math.sqrt(D)
    lo = torch.tensor([0] * 1 + [1] * 127 + [128] * 1 + [129] * 171)[:S]    # documents of 1, 127, 1, 171 tokens
    q, k, v = gen_seq(regime, H, D, S, lo, torch.arange(S), g, scale)
    return (q, k, v, lo, torch.arange(S), regime_slopes(regime, H), scale)


def _emulate(case, fam, **mistake):
    """Largest ratio of the mistaken reference over the correct one's bound, for ``out`` (or ``lse``)."""
    q, k, v, lo, hi, slopes, scale = case
    out, lse, p = attend(q, k, v, lo, hi, slopes, scale)
    atol, atol_lse = fwd_bounds(q, k, v, lo, hi, slopes, scale, out, lse, p, fam)
    args = dict(q=q, k=k, v=v, lo=lo, hi=hi, slopes=slopes, scale=scale, qpos=hi)
    what = mistake.pop("what", "out")
    args.update(mistake)
    bad_out, bad_lse, _ = attend(**args)
    if what == "lse":
        return _ratio(bad_lse * LOG2E, lse, atol_lse, 0.0)
    return _worst_ratio(bad_out, out, atol)


FLASH_MISTAKES = {
    # (regime, mistake on the reference's arguments)
    "causal_edge_one_key_too_wide": ("N", lambda c: dict(hi=c[4] + 1)),
    "causal_edge_one_key_too_narrow": ("R", lambda c: dict(hi=c[4] - 1, lo=torch.minimum(c[3], c[4] - 1))),
    "seg_start_one_key_too_wide": ("N", lambda c: dict(lo=(c[3] - 1).clamp_min(0))),
    "seg_start_one_key_too_narrow": ("N", lambda c: dict(lo=torch.minimum(c[3] + 1, c[4]))),
    "padded_width_softmax_scale": ("N", lambda c: dict(scale=1 / math.sqrt(128))),
    "neighbouring_heads_slope": ("R", lambda c: dict(slopes=c[5].roll(1))),
    "block_dropped": ("F", lambda c: dict(logw=torch.cat([torch.zeros(128), torch.full((128,), -math.inf),
                                                          torch.zeros(c[1].shape[1] - 256)]).double())),
}


@pytest.mark.parametrize("mistake", sorted(FLASH_MISTAKES))
def test_bounds_reject_flash_mistakes(mistake):
    regime, make = FLASH_MISTAKES[mistake]
    case = _flash_case(regime)
    r = _emulate(case, flash_family(64), **make(case))
    print(f"{mistake} ({regime}): largest |err| / bound = {r:.3g}")
    assert r > MARGIN


def test_bounds_reject_lse_in_log2_units():
    r = _emulate(_flash_case("R"), flash_family(64), what="lse")
    assert r > MARGIN


def _chunk_rescale_logw(case, c):
    """The weight 1 instead of exp2(m_c - M) for chunk c's partial: its keys scaled by exp(M - m_c)."""
    q, k, v, lo, hi, slopes, scale = case
    _, _, p = attend(q, k, v, lo, hi, slopes, scale)
    logp = torch.log(p)                                  # scores minus lse: the differences are what matters
    M = logp.max(-1, keepdim=True).values
    mc = logp[..., 64 * c:64 * c + 64].max(-1, keepdim=True).values
    w = torch.zeros_like(p)
    w[..., 64 * c:64 * c + 64] = torch.where(torch.isfinite(mc), M - mc, torch.zeros_like(mc)).expand(-1, -1, 64)
    return w


def _page_swapped(case, c):
    q, k, v, lo, hi, slopes, scale = case
    k, v = k.clone(), v.clone()
    k[:, 64 * c:64 * c + 64], v[:, 64 * c:64 * c + 64] = k[:, 64 * c + 64:64 * c + 128], v[:, 64 * c + 64:64 * c + 128]
    return dict(k=k, v=v)


DECODE_MISTAKES = {
    "lead_one_key_too_wide": ("N", 2, lambda c: dict(lo=c[3] - 1)),
    "lead_one_key_too_narrow": ("N", 1, lambda c: dict(lo=c[3] + 1)),
    "chunk_dropped": ("F", 0, lambda c: dict(logw=_chunk_logw(c[1].shape[1], 1, -math.inf))),
    "chunk_counted_twice": ("F", 0, lambda c: dict(logw=_chunk_logw(c[1].shape[1], 1, math.log(2.0)))),
    "chunk_merged_without_rescale": ("F", 0, lambda c: dict(logw=_chunk_rescale_logw(c, 1))),
    "page_read_through_neighbouring_entry": ("F", 0, lambda c: _page_swapped(c, 1)),
    "neighbouring_heads_slope": ("R", 0, lambda c: dict(slopes=c[5].roll(1))),
}


@pytest.mark.parametrize("L", [1000, 4097, 33000])
@pytest.mark.parametrize("mistake", sorted(DECODE_MISTAKES))
def test_bounds_reject_decode_mistakes(mistake, L):
    regime, first, make = DECODE_MISTAKES[mistake]
    lead = L // 3 if mistake.startswith("lead") else 0
    case = _decode_case(regime, L, lead=lead, first=first)
    r = _emulate(case, decode_family(64), **make(case))
    print(f"{mistake} ({regime}, L={L}): largest |err| / bound = {r:.3g}")
    assert r > MARGIN


@pytest.mark.parametrize("wide", [True, False])
def test_bounds_reject_append_query_offset(wide):
    """Append query j seeing pos + j + 1 (a leak, regime N) or pos + j - 1 (its own key dropped, regime R)."""
    regime = "N" if wide else "R"
    g = torch.Generator().manual_seed(13)
    D, H, pos, n = 64, 4, 1000, 8
    scale = 1 / math.sqrt(D)
    hi = torch.arange(pos, pos + n)
    q, k, v = gen_seq(regime, H, D, pos + n + 1, torch.zeros(n, dtype=torch.long), hi, g, scale)
    case = (q, k, v, torch.zeros(n, dtype=torch.long), hi, regime_slopes(regime, H), scale)
    r = _emulate(case, decode_family(64, unroll=2), hi=hi + (1 if wide else -1))
    assert r > MARGIN


@pytest.mark.parametrize("mistake", ["neighbouring_slots_scale", "new_token_from_decoy_slot"])
def test_bounds_reject_fp8_mistakes(mistake):
    """FP8 decode, regime R: the reference reads ``float(code) * scale`` before pos and qkv's token at pos."""
    g = torch.Generator().manual_seed(14)
    D, H, L = 64, 4, 1000
    scale = 1 / math.sqrt(D)
    q, k, v = gen_seq("R", H, D, L, torch.tensor([0]), torch.tensor([L - 1]), g, scale)
    (kc, ks), (vc, vs) = quantize_kv(k.float()), quantize_kv(v.float())
    deq = lambda c, s: c.double() * s.double().unsqueeze(-1)
    kr, vr = deq(kc, ks), deq(vc, vs)
    kr[:, -1], vr[:, -1] = k[:, -1], v[:, -1]
    case = (q, kr, vr, torch.tensor([0]), torch.tensor([L - 1]), regime_slopes("R", H), scale)
    if mistake == "neighbouring_slots_scale":
        kb, vb = deq(kc, ks.roll(-1, 1)), deq(vc, vs.roll(-1, 1))
        kb[:, -1], vb[:, -1] = k[:, -1], v[:, -1]
    else:
        dk, dv = decoy_rows(_bf(torch.randn(H, D, generator=g, dtype=torch.float64)))
        (dkc, dks), (dvc, dvs) = quantize_kv(dk.float()), quantize_kv(dv.float())
        kb, vb = kr.clone(), vr.clone()
        kb[:, -1], vb[:, -1] = deq(dkc, dks), deq(dvc, dvs)
    r = _emulate(case, decode_family(64, fp8=True), k=kb, v=vb)
    assert r > MARGIN


# ================================================================================================================
# GPU: the kernels against the float64 reference
# ================================================================================================================
FLASH_SHAPES = [(3, 1), (3, 2), (3, 17), (3, 127), (2, 128), (2, 129), (2, 1000), (1, 2049)]


def _flash_run(D, B, S, H, regime, seg, seed):
    """Forward (out and lse) and backward of the flash kernels on one layout, against the float64 reference."""
    from pipegoose_b200.ops import native
    g = torch.Generator().manual_seed(seed)
    scale = 1 / math.sqrt(D)
    slopes = regime_slopes(regime, H)
    segs = [torch.zeros(S, dtype=torch.long) if seg is None else seg[b].long() for b in range(B)]
    rows = []
    for b in range(B):
        q, k, v = gen_seq(regime, H, D, S, segs[b], torch.arange(S), g, scale)
        rows.append(torch.stack([q, k, v], 2).transpose(0, 1))              # [S, H, 3, D]
    qkv64 = torch.stack(rows).reshape(B * S, H * 3 * D)
    dout64 = _bf(torch.randn(B * S, H * D, generator=g, dtype=torch.float64))
    seg_dev = None if seg is None else seg.to(torch.int32).cuda()
    x = qkv64.to(torch.bfloat16).cuda().requires_grad_()
    sl = slopes.cuda()
    out = alibi_attention(x, sl, B, S, H, D, seg_start=seg_dev)
    out.backward(dout64.to(torch.bfloat16).cuda())
    DP = padded_head_dim(D)
    lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    out_p = torch.empty(B * S, H * DP, dtype=torch.bfloat16, device="cuda")
    native().attention_fwd(pad_heads(x.detach(), H, 3, D, DP).contiguous(), sl, out_p, lse, B, S, H, DP,
                           scale if DP != D else 0.0, None if seg_dev is None else seg_dev.reshape(-1))
    assert torch.equal(unpad_heads(out_p, H, 1, D, DP), out.detach())
    got_o, got_d = out.detach().view(B, S, H, D), x.grad.view(B, S, H, 3, D)
    fam = flash_family(D)
    tag = f"D{D}/{regime}"
    for b in range(B):
        xb = qkv64.view(B, S, H, 3, D)[b].cuda().transpose(0, 1)
        q, k, v = (xb[:, :, i].clone().requires_grad_() for i in range(3))
        lo, hi = segs[b].cuda(), torch.arange(S, device="cuda")
        o, l, p = attend(q, k, v, lo, hi, sl, scale)
        dO = dout64.view(B, S, H, D)[b].cuda().transpose(0, 1)
        o.backward(dO)
        grads = (q.grad, k.grad, v.grad)
        o, l, p = o.detach(), l.detach(), p.detach()
        q, k, v = q.detach(), k.detach(), v.detach()
        atol, atol_lse = fwd_bounds(q, k, v, lo, hi, sl, scale, o, l, p, fam)
        _check(f"flash_fwd/out/{tag}", got_o[b].transpose(0, 1), o, atol)
        _check(f"flash_fwd/lse/{tag}", lse[b], l, atol_lse, 0.0)
        _flash_bwd_checks(tag, q, k, v, hi, sl, scale, l, o, p, dO, grads, atol, atol_lse, got_d[b], S, D)


def _flash_bwd_checks(tag, q, k, v, hi, sl, scale, l, o, p, dO, grads, atol_o, atol_lse, got, S, D):
    """Backward bounds (module docstring) and checks of dQ, dK, dV for one row."""
    dq, dk, dv = grads
    j = torch.arange(S, device=q.device)
    s = torch.matmul(q, k.transpose(-1, -2)) * scale + sl.double().view(-1, 1, 1) * (j.view(1, 1, -1)
                                                                                   - hi.view(1, -1, 1)).double()
    qk = torch.matmul(q.abs(), k.abs().transpose(-1, -2)) * (scale * LOG2E)
    dist = (j.view(1, -1) - hi.view(-1, 1)).abs().double() + 128
    lse2 = (l * LOG2E).abs().unsqueeze(-1)
    dx = (D + 6) * U32 * qk + 3 * U32 * sl.double().abs().view(-1, 1, 1) * LOG2E * dist \
        + 2 * U32 * ((s * LOG2E).abs() + lse2) + U32 * lse2
    rho = torch.where(p > 0, LN2 * dx + atol_lse.unsqueeze(-1) + EXP_ERR, torch.zeros_like(p))
    dP = torch.matmul(dO, v.transpose(-1, -2))
    delta = (dO * o).sum(-1, keepdim=True)
    dS = p * (dP - delta) * scale
    d_delta = (dO.abs() * (atol_o + UBF * o.abs())).sum(-1, keepdim=True) + (D + 2) * U32 * (dO * o).abs().sum(-1, True)
    e_dP = (D + 6) * U32 * torch.matmul(dO.abs(), v.abs().transpose(-1, -2))
    e_dS = scale * (p * rho * (dP - delta).abs() + p * (d_delta + e_dP)) + (UBF + 2 * U32) * dS.abs()
    acc = (S + 4) * U32
    floor = (S + 4) * TINY * (1 + scale * (dP - delta).abs().max().item())      # underflow of tiny p
    atol_dv = torch.matmul((p * (rho + UBF)).transpose(-1, -2), dO.abs()) \
        + acc * torch.matmul(p.transpose(-1, -2), dO.abs()) + floor * dO.abs().max().item()
    atol_dk = torch.matmul(e_dS.transpose(-1, -2), q.abs()) + acc * torch.matmul(dS.abs().transpose(-1, -2), q.abs()) \
        + floor * q.abs().max().item()
    atol_dq = torch.matmul(e_dS, k.abs()) + acc * torch.matmul(dS.abs(), k.abs()) + floor * k.abs().max().item()
    for i, (name, want, atol) in enumerate((("dq", dq, atol_dq), ("dk", dk, atol_dk), ("dv", dv, atol_dv))):
        _check(f"flash_bwd/{name}/{tag}", got[:, :, i].transpose(0, 1), want, atol)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("B,S", FLASH_SHAPES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_flash_attention(D, B, S, regime):
    """Short rows with B > 1 put a partial query block over the next sequence's rows (``generate()``'s prefill)."""
    _flash_run(D, B, S, 2, regime, None, seed=D * 7 + S + B)


def _packed_seg():
    """Two rows of 600 tokens: documents of length 1 and documents starting at 127, 128, 129, 255, 256, 257, 385."""
    docs = [[1, 126, 1, 1, 128, 127, 1, 215], [129, 126, 1, 200, 144]]
    seg = []
    for row in docs:
        s, r = 0, []
        for n in row:
            r += [s] * n
            s += n
        seg.append(r)
    return torch.tensor(seg, dtype=torch.int32)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_flash_attention_packed(D, regime):
    _flash_run(D, 2, 600, 2, regime, _packed_seg(), seed=D + 3)


def _dec_check(name, got, q, k, v, lo, hi, slopes, scale, fam):
    out, lse, p = attend(q, k, v, lo, hi, slopes, scale)
    atol, _ = fwd_bounds(q, k, v, lo, hi, slopes, scale, out, lse, p, fam)
    _check(name, got, out, atol)


@gpu
@pytest.mark.parametrize("fill", ["nan", "decoy"])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_decode_attention(D, regime, fill):
    """The contiguous-cache decode kernel: every length, B = 3 with ``lead`` and B = 1 without; the slots before
    ``lead`` and from ``pos`` on hold NaN or decoy needles (the kernel writes slot ``pos``)."""
    H = 4
    scale = 1 / math.sqrt(D)
    slopes = regime_slopes(regime, H)
    fam = decode_family(D)
    for L in DEC_LENGTHS:
        g = torch.Generator().manual_seed(L + D)
        pos, cap = L - 1, L + 70
        for leads in ([0, min(1, pos), L // 3], None):
            rl = [0] if leads is None else leads
            qkv, kc, vc, seqs = _decode_layout(regime, H, D, cap, pos, rl, g, scale)
            hide = torch.ones(len(rl), 1, cap, 1, dtype=torch.bool)
            for b, l in enumerate(rl):
                hide[b, 0, min(l, pos):pos] = False
            if fill == "nan":
                kc, vc = kc.masked_fill(hide, math.nan), vc.masked_fill(hide, math.nan)
            else:
                dk, dv = decoy_rows(torch.stack([s[0][:, 0] for s in seqs]))          # [B, H, D]
                kc = torch.where(hide, dk.unsqueeze(2), kc)
                vc = torch.where(hide, dv.unsqueeze(2), vc)
            kd, vd = kc.to(torch.bfloat16).cuda(), vc.to(torch.bfloat16).cuda()
            lead_t = None if leads is None else torch.tensor(leads, dtype=torch.int32, device="cuda")
            out = alibi_decode_attention(qkv.to(torch.bfloat16).cuda(), kd, vd, slopes.cuda(), pos, lead_t, D)
            out = out.view(len(rl), H, D)
            for b, (q, k, v) in enumerate(seqs):
                _dec_check(f"decode/D{D}/{regime}", out[b].unsqueeze(1), q.cuda(), k.cuda(), v.cuda(),
                           torch.tensor([min(rl[b], pos)], device="cuda"), torch.tensor([pos], device="cuda"),
                           slopes.cuda(), scale, fam)


PAGED_GROUPS = [[1, 4097, 63], [2, 33000, 64], [65, 1000, 1], [33000]]


@gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("fill", ["nan", "decoy"])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_decode_attention(D, regime, fill, fp8):
    """The paged decode kernel over bf16 and FP8 pools: rows of every length over shuffled pages, unused slots NaN or
    decoy needles; over FP8 pools the reference reads ``float(code) * scale`` before ``pos`` and qkv's token at it."""
    H = 4
    scale = 1 / math.sqrt(D)
    slopes = regime_slopes(regime, H)
    fam = decode_family(D, fp8=fp8)
    for gi, lengths in enumerate(PAGED_GROUPS):
        g = torch.Generator().manual_seed(D + 100 * gi)
        seqs = [gen_seq(regime, H, D, n + 1, torch.tensor([0]), torch.tensor([n - 1]), g, scale, first=b)
                for b, n in enumerate(lengths)]
        pools, table, kf, vf = build_pools(seqs, lengths, H, D, fill, g, fp8=fp8, dev="cuda",
                                           stored=[n - 1 for n in lengths])
        B = len(lengths)
        qkv = torch.stack([torch.stack([q[:, 0], k[:, n - 1], v[:, n - 1]], 1)
                           for (q, k, v), n in zip(seqs, lengths)]).view(B, H * 3 * D)
        pos = torch.tensor([n - 1 for n in lengths], dtype=torch.int32, device="cuda")
        kw = dict(k_scales=pools[2], v_scales=pools[3]) if fp8 else {}
        out = alibi_paged_decode_attention(qkv.to(torch.bfloat16).cuda(), pools[0], pools[1], table, pos,
                                           max(lengths) - 1, slopes.cuda(), D, **kw).view(B, H, D)
        kf, vf = kf.cuda(), vf.cuda()
        for b, ((q, k, v), n) in enumerate(zip(seqs, lengths)):
            kk, vv = paged_rows(kf, table[b], n), paged_rows(vf, table[b], n)
            kk[:, n - 1], vv[:, n - 1] = k[:, n - 1].cuda(), v[:, n - 1].cuda()
            _dec_check(f"paged_decode{'_fp8' if fp8 else ''}/D{D}/{regime}", out[b].unsqueeze(1), q.cuda(), kk, vv,
                       torch.tensor([0], device="cuda"), torch.tensor([n - 1], device="cuda"), slopes.cuda(), scale,
                       fam)


APPEND_CACHED = [0, 1, 63, 64, 65, 1000, 4097, 33000]


@gpu
@pytest.mark.parametrize("most", [1, 2, 4, 8])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_append_attention(D, regime, most):
    """The append kernel at every query tile: rows of 1 .. ``most`` tokens over every cached length; unused slots NaN
    for tiles 1 and 4, decoy needles for tiles 2 and 8."""
    H = 4
    scale = 1 / math.sqrt(D)
    slopes = regime_slopes(regime, H)
    fill = "nan" if most in (1, 4) else "decoy"
    g = torch.Generator().manual_seed(D + most)
    news = [i % most + 1 for i in range(len(APPEND_CACHED))]
    qkv, pools, table, cu, st, refs = _append_layout(regime, H, D, APPEND_CACHED, news, fill, g, scale, dev="cuda")
    max_pos = max(s + n - 1 for s, n in zip(APPEND_CACHED, news))
    out = alibi_paged_append_attention(qkv.to(torch.bfloat16).cuda(), pools[0], pools[1], table, cu.cuda(), st.cuda(),
                                       max_pos, slopes.cuda(), D, max_tokens=most).view(-1, H, D)
    fam = decode_family(D, unroll=4 if most <= 2 else 2)
    for r, ref in enumerate(refs):
        ref = tuple(t.cuda() for t in ref)
        _dec_check(f"append/D{D}/{regime}", out[int(cu[r]):int(cu[r + 1])].transpose(0, 1), *ref, slopes.cuda(),
                   scale, fam)


STARTS = [0, 64, 1000, 4160]
FP8_STARTS = [0, 64, 1024, 4160]
NEWS = [1, 2, 127, 128, 129, 1000]


@gpu
@pytest.mark.parametrize("fp8", [False, pytest.param(True, id="fp8_staged")])
@pytest.mark.parametrize("fill", ["nan", "decoy"])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("D", [64, 80, 128])
def test_paged_prefill_attention(D, regime, fill, fp8):
    """The paged prefill kernel over bf16 pools (every position in the pools) and over FP8 pools through a staging pool
    (cached positions dequantized from the FP8 pools, new ones from qkv), every start with every number of new
    tokens."""
    H = 4
    scale = 1 / math.sqrt(D)
    slopes = regime_slopes(regime, H)
    g = torch.Generator().manual_seed(D + 7 * fp8)
    rows = [(s, n) for s in (FP8_STARTS if fp8 else STARTS) for n in NEWS]
    starts, news = [r[0] for r in rows], [r[1] for r in rows]
    qkv, pools, table, cu, st, refs = _prefill_layout(regime, H, D, starts, news, fill, g, scale, fp8=fp8, dev="cuda")
    kw = {}
    if fp8:
        lengths = [s + n for s, n in zip(starts, news)]
        pages = [table[r, :-(-n // PAGE_SIZE)].tolist() for r, n in enumerate(lengths)]
        num, src, dst, slot, st_table = fp8_prefill_staging(pages, starts, lengths)
        k_stage = torch.full((num, H, PAGE_SIZE, D), math.nan, dtype=torch.bfloat16, device="cuda")
        dev = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
        kw = dict(k_scales=pools[2], v_scales=pools[3],
                  stage=(k_stage, k_stage.clone(), dev(src), dev(dst), dev(slot), dev(st_table)))
    out = alibi_paged_prefill_attention(qkv.to(torch.bfloat16).cuda(), pools[0], pools[1], table, cu.cuda(),
                                        st.cuda(), max(news), slopes.cuda(), D, **kw).view(-1, H, D)
    fam = flash_family(D)
    for r, ref in enumerate(refs):
        ref = tuple(t.cuda() for t in ref)
        _dec_check(f"paged_prefill{'_fp8' if fp8 else ''}/D{D}/{regime}",
                   out[int(cu[r]):int(cu[r + 1])].transpose(0, 1), *ref, slopes.cuda(), scale, fam)
