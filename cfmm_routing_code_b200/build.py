"""Build libcfmm_b200.so in-tree with nvcc for sm_90a (H100; no torch dependency: plain C ABI)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, os.environ.get("CFMM_LIB", "libcfmm_b200.so"))      # (CFMM_LIB: load / build an experiment variant)
SOURCES = ["cfmm_kernels.cu", "cfmm_blocked.cu", "cfmm_layout.cu", "cfmm_persist.cu", "cfmm_solver.cu", "cfmm_allreduce.cu",
           "cfmm_small.cu", "cfmm_small_ladder.cu", "cfmm_splice.cu", "cfmm_small_crypto.cu",
           "cfmm_small_tricrypto.cu", "cfmm_small_bins.cu", "cfmm_small_eclp.cu", "cfmm_small_pmm.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA path cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    if os.environ.get("CFMM_LIB"):          # an experiment variant built by hand (its -D flags are not known here): use as is
        return False
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "cfmm_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile every translation unit to an object in parallel (each one is compiled whole, as a single nvcc call
    would; ptxas runs single-threaded per unit, and the per-thread solver instances take it minutes), then link the
    shared library.  The ptxas report of every unit, in SOURCES order, goes to build_ptxas.log."""
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    extra = os.environ.get("CFMM_NVCC_EXTRA", "").split()
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC]
    with tempfile.TemporaryDirectory(prefix="cfmm_build_") as tmp:
        objs = [os.path.join(tmp, os.path.splitext(s)[0] + ".o") for s in SOURCES]

        def compile_one(k):
            cmd = [nvcc] + NVCC_FLAGS + extra + inc + ["-c", os.path.join(CSRC, SOURCES[k]), "-o", objs[k]]
            return subprocess.run(cmd, capture_output=True, text=True)
        with ThreadPoolExecutor(max_workers=max(1, min(len(SOURCES), os.cpu_count() or 1))) as ex:
            results = list(ex.map(compile_one, range(len(SOURCES))))
        log = "".join(r.stdout + r.stderr for r in results)
        failed = [s for s, r in zip(SOURCES, results) if r.returncode != 0]
        link = None
        if not failed:
            link = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                                   "-o", LIB] + objs, capture_output=True, text=True)
            log += link.stdout + link.stderr
        if verbose or failed or link.returncode != 0:
            sys.stderr.write(log)
        if failed or link.returncode != 0:
            raise RuntimeError("nvcc failed building libcfmm_b200.so" + (f" ({', '.join(failed)})" if failed else ""))
    with open(os.path.join(HERE, "build_ptxas.log"), "w") as f:
        f.write(log)
    return LIB


if __name__ == "__main__":
    print(build_library(force=True, verbose="-v" in sys.argv))
