"""In-tree build of the sm_90a extension ``pipegoose_b200/_C*.so``.

Every ``*.cu`` under ``csrc/`` is compiled straight by nvcc with
``-gencode arch=compute_90a,code=sm_90a -lineinfo`` (no torch headers, so a kernel file
rebuilds in seconds); ``bindings.cpp`` is the only translation unit that sees torch.  Objects
are cached under ``csrc/build/`` keyed by a content hash of the source and the headers.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent
PKG = CSRC.parent
BUILD = CSRC / "build"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + [
    "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


# PIPEGOOSE_B200_BUILD_VARIANT=<name> + PIPEGOOSE_B200_NVCC_EXTRA="-DFOO=1 ...": build pipegoose_b200/_C_<name>.so with extra
# nvcc flags next to the main extension (loaded with PIPEGOOSE_B200_EXT=<name>): A/B of kernel variants in one process
VARIANT = os.environ.get("PIPEGOOSE_B200_BUILD_VARIANT", "")
NVCC_FLAGS = NVCC_FLAGS + os.environ.get("PIPEGOOSE_B200_NVCC_EXTRA", "").split()
if VARIANT:
    BUILD = CSRC / f"build_{VARIANT}"


def so_path() -> Path:
    return PKG / (f"_C_{VARIANT}.so" if VARIANT else "_C.so")


def _hash(paths) -> str:
    h = hashlib.sha1()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def _run(cmd, log: Path | None = None):
    res = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        log.write_text(res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("command failed: " + " ".join(map(str, cmd)))
    return res


def build(verbose: bool = False, force: bool = False) -> Path:
    import torch
    from torch.utils import cpp_extension as ce

    BUILD.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
    cus = sorted(CSRC.glob("*.cu"))
    objs = []
    jobs = []
    for cu in cus:
        tag = _hash([cu] + headers)
        obj = BUILD / f"{cu.stem}.{tag}.o"
        objs.append(obj)
        if force or not obj.exists():
            for old in BUILD.glob(f"{cu.stem}.*.o"):
                old.unlink()
            jobs.append((cu, obj))

    def compile_cu(job):
        cu, obj = job
        if verbose:
            print(f"[pipegoose_b200] nvcc {cu.name}", flush=True)
        _run([NVCC, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(cu), "-o", str(obj)],
             log=BUILD / f"{cu.stem}.ptxas.log")

    # bindings (torch headers; g++)
    bind_src = CSRC / "bindings.cpp"
    bind_tag = _hash([bind_src] + headers)
    bind_obj = BUILD / f"bindings.{bind_tag}.o"
    need_bind = force or not bind_obj.exists()

    def compile_bind(_):
        if verbose:
            print("[pipegoose_b200] g++ bindings.cpp", flush=True)
        for old in BUILD.glob("bindings.*.o"):
            old.unlink()
        inc = []
        for p in ce.include_paths():
            inc += ["-isystem", p]
        inc += ["-isystem", sysconfig.get_paths()["include"], "-isystem", "/usr/local/cuda/include"]
        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
        _run(["g++", "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
              "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
              *inc, "-I", str(CSRC), "-c", str(bind_src), "-o", str(bind_obj)])

    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as ex:
        futs = [ex.submit(compile_cu, j) for j in jobs]
        if need_bind:
            futs.append(ex.submit(compile_bind, None))
        for f in futs:
            f.result()

    out = so_path()
    stamp = BUILD / "link.stamp"
    link_tag = "|".join(o.name for o in objs + [bind_obj])
    if force or jobs or need_bind or not out.exists() or not stamp.exists() or stamp.read_text() != link_tag:
        torch_lib = ce.library_paths()[0]
        cmd = [NVCC, "-shared", "-o", str(out), *map(str, objs), str(bind_obj),
               *ARCH_FLAGS, "-L", torch_lib, "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python",
               "-lc10_cuda", "-ltorch_cuda", "-Xlinker", f"-rpath={torch_lib}"]
        _run(cmd)
        stamp.write_text(link_tag)
        if verbose:
            print(f"[pipegoose_b200] linked {out}", flush=True)
    return out


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
