"""``python -m pipegoose_b200`` — what this installation can do on this machine (paste it into a bug report).

Prints the package / torch / CUDA versions, whether the sm_90a extension is built and loads, the GPUs and whether they can
address each other's memory (the NVLink engines need peer access), the ``PIPEGOOSE_B200_*`` switches that are set, and the
launcher environment.  Never raises: every probe that fails is reported as such.
"""
from __future__ import annotations

import os
import sys


def _probe(label, fn):
    try:
        value = fn()
    except Exception as e:  # a report tool must not die on the thing it reports
        value = f"FAILED: {type(e).__name__}: {e}"
    print(f"{label:<28} {value}")
    return value


def main() -> int:
    import torch

    import pipegoose_b200

    root = os.path.dirname(os.path.abspath(pipegoose_b200.__file__))
    _probe("pipegoose_b200", lambda: f"{pipegoose_b200.__version__} ({root})")
    _probe("python / torch", lambda: f"{sys.version.split()[0]} / {torch.__version__} (CUDA {torch.version.cuda})")
    so = os.path.join(root, "_C.so")
    _probe("extension (_C.so)", lambda: f"built, {os.path.getsize(so) / 2**20:.1f} MiB" if os.path.exists(so)
           else "NOT BUILT: python -m pipegoose_b200.csrc.build (nvcc, no GPU needed)")
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    _probe("GPUs", lambda: f"{n}" + (": " + ", ".join(sorted({torch.cuda.get_device_name(i) for i in range(n)})) if n else
                                     " (CPU only: gloo paths and PyTorch fallbacks of every op)"))
    if n:
        _probe("compute capability", lambda: ", ".join(sorted({"sm_%d%d" % torch.cuda.get_device_capability(i) for i in range(n)}))
               + "  (the kernels are sm_90a only)")
        _probe("extension loads", lambda: sorted(k for k in dir(__import__("pipegoose_b200.ops", fromlist=["native"]).native())
                                                  if not k.startswith("_"))[:4] + ["..."])
        if n > 1:
            _probe("peer access (NVLink engines)", lambda: "all pairs" if all(
                torch.cuda.can_device_access_peer(i, j) for i in range(n) for j in range(n) if i != j) else "NOT all pairs")
        _probe("NCCL", lambda: ".".join(map(str, torch.cuda.nccl.version())))
    _probe("distributed backends", lambda: ", ".join(b for b in ("nccl", "gloo", "mpi")
                                                     if getattr(torch.distributed, f"is_{b}_available")()))
    switches = {k: v for k, v in sorted(os.environ.items()) if k.startswith("PIPEGOOSE_B200_")}
    _probe("switches set", lambda: switches or "none (defaults: docs/CONFIGURATION.md)")
    launcher = {k: os.environ[k] for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT",
                                           "TORCHELASTIC_RESTART_COUNT") if k in os.environ}
    _probe("launcher environment", lambda: launcher or "not under torchrun")
    repo = os.path.dirname(root)
    _probe("reference arm (bench)", lambda: "installed" if os.path.isdir(os.path.join(repo, "baseline", "_ref", "pipegoose"))
           else "not installed (DESIGN.md §4)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
