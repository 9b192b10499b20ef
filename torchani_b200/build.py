"""In-tree build of the C-ABI library ``libani_b200.so`` (nvcc, sm_90a only).

The library has no torch / python dependency: plain ``extern "C"`` entry points declared in
``include/ani_b200.h``.  ``python -m torchani_b200.build`` (or ``__graft_entry__.build()``)
compiles every ``csrc/*.cu`` and links them next to this file.

Variants: the default library uses 2 x fp16 GEMM operand pieces; ``build(variant="bf16x3")``
(``python -m torchani_b200.build --variant bf16x3``) compiles the same sources with
``-DANI_OPND_FP16X2=0`` into ``libani_b200_bf16x3.so`` (select it with ``ANI_B200_LIB=<path>``).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "csrc", "build")
LIB = os.path.join(HERE, "libani_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


VARIANTS = {
    "": [],
    "bf16x3": ["-DANI_OPND_FP16X2=0"],
    # tuning experiments (occupancy of the AEV kernels); not built by default
    "bwd5": ["-DANI_AEV_BWD_MIN_CTAS=5"],
    "bwd6": ["-DANI_AEV_BWD_MIN_CTAS=6"],
    "fwd7": ["-DANI_AEV_FWD_MIN_CTAS=7", "-DANI_AEV_CAND_CAP=640"],
    "fwd8w": ["-DANI_AEV_FWD_WARPS=8", "-DANI_AEV_FWD_MIN_CTAS=3"],
    "fwd6w": ["-DANI_AEV_FWD_WARPS=6", "-DANI_AEV_FWD_MIN_CTAS=4"],
    # phase trace of the CTA-staged AEV forward (tools/aev_forward_trace.py)
    "aevtrace": ["-DANI_AEV_FWD_TRACE=1"],
}


def lib_path(variant: str = "") -> str:
    return LIB if not variant else os.path.join(HERE, f"libani_b200_{variant}.so")


def _fingerprint(extra=()) -> str:
    h = hashlib.sha256()
    files = _sources() + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    files.append(os.path.join(os.path.dirname(HERE), "include", "ani_b200.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(list(NVCC_FLAGS) + list(extra)).encode())
    return h.hexdigest()


# translation units without any of the profiled kernels (preparation, communicator, pair potentials, dispersion, ABI
# glue, Hessians, MD integrators, FIRE, L-BFGS, NEB): a change there does not touch the AEV / GEMM kernels whose measured DRAM traffic bench.py reports
_NOT_PROFILED = ("cells.cu", "comm.cu", "api.cu", "pair.cu", "disp.cu", "charges.cu", "hessian.cu", "md.cu",
                "opt.cu", "lbfgs.cu", "neb.cu")


def build_id(variant: str = "", kernels_only: bool = False) -> str:
    """Identity of the library build on disk: the fingerprint of the sources + flags it was compiled from (nvcc output
    is not byte-reproducible, the sources are), or "" when the library is missing or older than the sources.
    ``kernels_only``: the fingerprint of what the AEV and GEMM kernels are compiled from (``aev.cu``, ``mlp.cu``, the
    headers, the flags) -- the key of profiles/traffic.json."""
    bdir = BUILD if not variant else BUILD + "_" + variant
    stamp = os.path.join(bdir, "fingerprint.txt")
    if not (os.path.exists(lib_path(variant)) and os.path.exists(stamp)):
        return ""
    fp = _fingerprint(VARIANTS[variant])
    if open(stamp).read() != fp:
        return ""
    if not kernels_only:
        return fp[:16]
    h = hashlib.sha256()
    files = [f for f in _sources() if os.path.basename(f) not in _NOT_PROFILED]
    files += [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    files.append(os.path.join(os.path.dirname(HERE), "include", "ani_b200.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(list(NVCC_FLAGS) + list(VARIANTS[variant])).encode())
    return "k" + h.hexdigest()[:15]


def build(force: bool = False, verbose: bool = False, variant: str = "") -> str:
    extra = VARIANTS[variant]
    bdir = BUILD if not variant else BUILD + "_" + variant
    lib = lib_path(variant)
    os.makedirs(bdir, exist_ok=True)
    stamp = os.path.join(bdir, "fingerprint.txt")
    fp = _fingerprint(extra)
    if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == fp:
        return lib
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(bdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(bdir, os.path.basename(src)[:-3] + ".ptxas.log")
        with open(log, "w") as fh:
            fh.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            print(res.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [nvcc, "-shared", "--cudart", "shared", "-o", lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    with open(stamp, "w") as fh:
        fh.write(fp)
    return lib


if __name__ == "__main__":
    _variant = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else ""
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=_variant))
