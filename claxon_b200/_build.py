"""In-tree builds of the native pieces (no JIT cache: the .so files travel with the tree).

* ``libclaxon_b200.so`` — the product: CUDA kernels for sm_90a (H100) + the C ABI of
  ``include/claxon_b200.h`` + the C++ host side (demux, header parse, facade).
* ``libclxsynth.so``    — the synthetic frame generator (plain C, host only).
"""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libclaxon_b200.so")
SYNTH = os.path.join(HERE, "libclxsynth.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall", "-shared", "--use_fast_math", "-Xptxas", "-v",
]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(s) and os.path.getmtime(s) > t for s in sources)


def lib_sources() -> list[str]:
    names = sorted(os.listdir(CSRC))
    return [os.path.join(CSRC, n) for n in names if n.endswith((".cu", ".cpp"))]


def lib_deps() -> list[str]:
    deps = [os.path.join(CSRC, n) for n in os.listdir(CSRC)]
    inc = os.path.join(ROOT, "include")
    deps += [os.path.join(inc, n) for n in os.listdir(inc)]
    return deps


def nvcc_path() -> str | None:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """Compiles the CUDA extension for sm_90a with nvcc (cross-compiles without a GPU).

    CLX_EXPERIMENT=1 builds and selects ``libclaxon_b200_exp.so`` instead: the same sources with the
    measurement switches of tools/exp_*.py compiled in (-DCLX_EXPERIMENT); the product library has none."""
    global LIB
    if os.environ.get("CLX_EXPERIMENT"):
        LIB = os.path.join(HERE, "libclaxon_b200_exp.so")
    if os.environ.get("CLX_RING_TMA"):
        LIB = LIB.replace(".so", "_tma.so")
    if os.environ.get("CLX_DEC_WARPS"):
        LIB = LIB.replace(".so", "_w" + str(int(os.environ["CLX_DEC_WARPS"])) + ".so")
    if not force and not _newer(LIB, lib_deps()):
        return LIB
    nvcc = nvcc_path()
    if nvcc is None:
        if os.path.exists(LIB):
            return LIB  # a machine without the CUDA toolkit: use the library built elsewhere
        raise RuntimeError("nvcc not found and no prebuilt libclaxon_b200.so")
    extra = []
    if os.environ.get("CLX_EXPERIMENT"):
        extra.append("-DCLX_EXPERIMENT")
    if os.environ.get("CLX_RING_TMA"):
        extra.append("-DCLX_RING_TMA")
    if os.environ.get("CLX_DEC_WARPS"):
        extra.append("-DCLX_DEC_WARPS=" + str(int(os.environ["CLX_DEC_WARPS"])))
    cmd = [nvcc, *NVCC_FLAGS, *extra, "-I", os.path.join(ROOT, "include"), "-o", LIB, *lib_sources()]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if verbose:
        print(log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-4000:])
    return LIB


def build_synth(force: bool = False) -> str:
    src = os.path.join(CSRC, "synth.c")
    if not force and not _newer(SYNTH, [src]):
        return SYNTH
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        if os.path.exists(SYNTH):
            return SYNTH
        raise RuntimeError("gcc not found and no prebuilt libclxsynth.so")
    subprocess.check_call([gcc, "-O2", "-fPIC", "-shared", "-o", SYNTH, src, "-lm", "-lpthread"])
    return SYNTH
