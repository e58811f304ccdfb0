"""CPU checks of FP8 training (``BloomConfig(fp8=True)``): the reference quantizer that defines the cast kernels' format,
and the configurations the FP8 blocks refuse.  The kernels themselves are checked in ``test_gpu_fp8_training.py``."""
import numpy as np
import pytest
import torch
from torch import nn

from pipegoose_b200.models.bloom import BloomConfig, BloomForCausalLM
from pipegoose_b200.ops.kernels import FP8_FORMATS, fp8_quantize_reference

FMTS = ["e4m3", "e5m2"]


def _finite_codes(dtype):
    """Every finite non-negative value of the format, ascending, with its code."""
    codes = torch.arange(256, dtype=torch.uint8)
    vals = codes.view(dtype).float()
    keep = torch.isfinite(vals) & (vals >= 0) & (codes < 128)
    vals, codes = vals[keep], codes[keep]
    order = torch.argsort(vals)
    return vals[order], codes[order]


@pytest.mark.parametrize("fmt", FMTS)
def test_scale_formula(fmt):
    dtype, fmax = FP8_FORMATS[fmt]
    torch.manual_seed(0)
    x = (torch.randn(37, 24) * 3.7).to(torch.bfloat16)
    codes, scale_inv = fp8_quantize_reference(x, fmt)
    amax = np.float32(x.float().abs().max().item())
    assert codes.dtype == dtype and codes.shape == x.shape
    assert scale_inv.dtype == torch.float32 and scale_inv.shape == (1,)
    assert scale_inv.item() == np.float32(amax / np.float32(fmax))          # IEEE fp32 division
    scale = np.float32(np.float32(fmax) / amax)
    want = torch.from_numpy(np.clip(x.float().numpy() * scale, -fmax, fmax)).to(dtype)
    assert torch.equal(codes.view(torch.uint8), want.view(torch.uint8))
    # the largest |x| lands on fmax (or one rounding step below it), nothing saturates beyond
    assert codes.float().abs().max().item() <= fmax
    assert codes.float().abs().max().item() >= fmax * (1 - 2.0 ** -3)
    # dequantized values are x to the format's relative precision
    err = (codes.float() * scale_inv - x.float()).abs()
    u = 2.0 ** -4 if fmt == "e4m3" else 2.0 ** -3
    assert bool((err <= u * x.float().abs() + 2.0 ** -9 * amax).all())


@pytest.mark.parametrize("fmt", FMTS)
def test_zero_tensor(fmt):
    codes, scale_inv = fp8_quantize_reference(torch.zeros(8, 16, dtype=torch.bfloat16), fmt)
    assert scale_inv.item() == 1.0
    assert bool((codes.view(torch.uint8) == 0).all())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_non_finite_amax_gives_nan_scale_inv(fmt, bad):
    x = torch.randn(8, 16).to(torch.bfloat16)
    x[3, 5] = bad
    _, scale_inv = fp8_quantize_reference(x, fmt)
    assert torch.isnan(scale_inv).all(), "a non-finite amax must not turn into a finite scale"


@pytest.mark.parametrize("fmt", FMTS)
def test_torch_float8_cast_is_round_to_nearest_even(fmt):
    """Within range, the reference's ``.to(float8)`` is round-to-nearest-even onto the format's grid: every midpoint of
    two neighbouring values goes to the one with the even code, and the fp32 values next to it to the nearer one.
    Beyond ``fmax`` the reference clamps first (the kernels' ``satfinite``)."""
    dtype, fmax = FP8_FORMATS[fmt]
    vals, codes = _finite_codes(dtype)
    assert vals[-1].item() == fmax
    lo, hi = vals[:-1].numpy(), vals[1:].numpy()
    mid = ((lo.astype(np.float64) + hi) / 2).astype(np.float32)
    assert np.all((mid.astype(np.float64) * 2) == lo.astype(np.float64) + hi)     # exact in fp32
    even = np.where(codes[:-1].numpy() % 2 == 0, lo, hi)
    below = np.nextafter(mid, np.float32(-np.inf))
    above = np.nextafter(mid, np.float32(np.inf))
    for sign in (1.0, -1.0):
        for inp, want in ((mid, even), (below, lo), (above, hi), (lo, lo)):
            got = torch.from_numpy(sign * inp).to(dtype).float().numpy()
            assert np.array_equal(got, sign * want)
    big = torch.tensor([fmax * 1.01, 1e30, float("inf"), -fmax * 1.5])
    assert torch.clamp(big, -fmax, fmax).to(dtype).float().tolist() == [fmax, fmax, fmax, -fmax]


def _tiny(**kw):
    return BloomForCausalLM(BloomConfig(vocab_size=64, hidden_size=32, n_layer=1, n_head=2, fp8=True, **kw))


def _run(model):
    ids = torch.randint(0, 64, (2, 16))
    return model(ids, labels=ids)


def test_fp8_is_off_by_default():
    assert BloomConfig().fp8 is False
    from pipegoose_b200.models.gpt2 import GPT2Config

    assert GPT2Config(fp8=True).fp8 is True


def test_fp8_refuses_the_cpu_fp32_path():
    with pytest.raises(ValueError, match="native path"):
        _run(_tiny())


def test_fp8_refuses_tensor_parallelism():
    model = _tiny()
    model.transformer.h[0].tp = object()
    with pytest.raises(ValueError, match="tensor parallelism"):
        _run(model)


def test_fp8_refuses_dropout_in_training():
    model = _tiny(hidden_dropout=0.1)
    model.train()
    with pytest.raises(ValueError, match="dropout"):
        _run(model)


def test_fp8_refuses_a_replaced_mlp():
    class Experts(nn.Module):
        def forward(self, hidden_states, residual):
            return hidden_states + residual

    model = _tiny()
    model.transformer.h[0].mlp = Experts()
    with pytest.raises(ValueError, match="Experts"):
        _run(model)
