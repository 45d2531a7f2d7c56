"""Builds libdiartb200.so (sm_90a) in-tree with nvcc; no CPU fallback exists.

    python -m diart_b200.build          # or diart_b200.build.build()
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libdiartb200.so")
SOURCES = ["api.cu", "api_seg.cu", "api_emb.cu", "api_cluster.cu", "api_stream.cu", "api_post.cu", "api_pipeline.cu", "api_multi.cu",
           "sincnet.cu", "gemm.cu", "gemm_tc.cu", "sinc_tc.cu", "lstm_tc.cu", "heads.cu", "cluster.cu", "post.cu", "resnet.cu", "resample.cu", "der.cu",
           "vad.cu", "api_gallery.cu", "gallery.cu", "transfer.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def have_nvcc() -> bool:
    return any(c and os.path.exists(c) for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"))


HASH = OUT + ".hash"


def _source_hash() -> str:
    import hashlib

    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(HERE, "..", "include", "diart_b200.h")]
    for path in files:
        if os.path.isfile(path):
            h.update(os.path.basename(path).encode())
            h.update(open(path, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _stale() -> bool:
    """content hash of the sources vs the one recorded at build time (time stamps do not survive a copy to another box)"""
    if not os.path.exists(OUT) or not os.path.exists(HASH):
        return True
    return open(HASH).read().strip() != _source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", OUT, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcuda"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(HASH, "w") as f:
        f.write(_source_hash() + "\n")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
