"""Python front-end of the sm_90a kernels.

``native()`` returns the in-tree extension module (``pipegoose_b200/_C.so``, built by
``pipegoose_b200/csrc/build.py``).  On a machine with a CUDA device the extension is mandatory:
ops raise instead of silently falling back to eager PyTorch.  On CPU-only machines (unit tests
with gloo) the ops use reference PyTorch math.
"""
from __future__ import annotations

import importlib.util
import os
from pathlib import Path

import torch

_C = None
_LOAD_ERROR = None


def _load():
    global _C, _LOAD_ERROR
    if _C is not None or _LOAD_ERROR is not None:
        return
    # PIPEGOOSE_B200_EXT=<name>: load a variant build (pipegoose_b200/_C_<name>.so, made with PIPEGOOSE_B200_BUILD_VARIANT=<name>
    # PIPEGOOSE_B200_NVCC_EXTRA="-D..." python -m pipegoose_b200.csrc.build) instead of the main one — lets ONE GPU call A/B
    # kernel variants under identical Python
    variant = os.environ.get("PIPEGOOSE_B200_EXT", "")
    so = Path(__file__).resolve().parent.parent / (f"_C_{variant}.so" if variant else "_C.so")
    if variant and not so.exists():
        _LOAD_ERROR = FileNotFoundError(f"{so} not found: build it with PIPEGOOSE_B200_BUILD_VARIANT={variant} (csrc/build.py)")
        return
    if not so.exists():
        if os.environ.get("PIPEGOOSE_B200_AUTOBUILD", "0") == "1":
            from pipegoose_b200.csrc.build import build

            build()
        else:
            _LOAD_ERROR = FileNotFoundError(
                f"{so} not found: build it with `python -m pipegoose_b200.csrc.build` "
                "(or `python -c 'import __graft_entry__ as g; g.build()'`)"
            )
            return
    try:
        spec = importlib.util.spec_from_file_location("pipegoose_b200._C", so)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _C = mod
    except Exception as e:  # pragma: no cover
        _LOAD_ERROR = e


# kernels launched per binding call (everything else launches exactly one)
_LAUNCHES_PER_CALL = {"layernorm_bwd": 2, "attention_bwd": 3}  # dx + params; delta + bwd + dQ convert
_launch_count = 0
_PROXY = None


class _CountingProxy:
    """Forwards to the extension and counts the kernels it launches (bench.py's ``gpu_launches``)."""

    def __init__(self, mod):
        self._mod = mod

    def __getattr__(self, name):
        fn = getattr(self._mod, name)
        n = _LAUNCHES_PER_CALL.get(name, 1)

        def wrapped(*a, **k):
            global _launch_count
            _launch_count += n
            return fn(*a, **k)

        wrapped.__name__ = name
        self.__dict__[name] = wrapped
        return wrapped


def native():
    """The compiled extension, or raise with the reason it is unavailable."""
    global _PROXY
    if _PROXY is None:
        _load()
        if _C is None:
            raise RuntimeError(f"pipegoose_b200 native extension unavailable: {_LOAD_ERROR}")
        _PROXY = _CountingProxy(_C)
    return _PROXY


def reset_launch_count():
    global _launch_count
    _launch_count = 0


def launch_count() -> int:
    return _launch_count


def have_native() -> bool:
    _load()
    return _C is not None


def has_kernel(name: str) -> bool:
    return have_native() and hasattr(_C, name)


def use_native(*tensors) -> bool:
    """True when the op must run on the sm_90a kernels (CUDA bf16 inputs).

    Raises if CUDA tensors are given but the extension is missing: a GPU run never degrades to
    an eager fallback silently.
    """
    t = next((t for t in tensors if isinstance(t, torch.Tensor)), None)
    if t is None or not t.is_cuda:
        return False
    if t.dtype != torch.bfloat16:
        return False
    native()
    return True
