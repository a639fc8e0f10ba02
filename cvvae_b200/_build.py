"""In-tree build of libcvvae_b200.so (nvcc, sm_90a only).

The shared object lands in ``cvvae_b200/lib/`` inside the tree, so the package imports from the repository;
nothing is installed into site-packages and no JIT cache is used.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBPATH = os.path.join(LIBDIR, "libcvvae_b200.so")
SOURCES = ["api.cu", "conv_tc.cu", "conv_stk.cu", "conv_direct.cu", "groupnorm.cu", "attention.cu", "misc.cu", "video_io.cu",
           "metrics.cu", "lpips.cu", "i3d.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; cannot build libcvvae_b200.so")
    return cand


def _stale() -> bool:
    if not os.path.exists(LIBPATH):
        return True
    t = os.path.getmtime(LIBPATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), "include", "cvvae_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a and link the C-ABI shared library. Returns its path."""
    if not force and not _stale():
        return LIBPATH
    nvcc = _nvcc()
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src: str) -> str:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    tmp = LIBPATH + ".tmp"
    r = subprocess.run([nvcc, "-shared", "-cudart", "static", "-o", tmp, *objs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIBPATH)
    return LIBPATH


if __name__ == "__main__":
    print(build_library(force=True, verbose=True))
