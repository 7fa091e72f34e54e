"""Builds libgsql_gpu.so (the C-ABI shared library) in-tree with nvcc for sm_90a (H100).

No GPU is needed to build (nvcc cross-compiles).  The .so lands in galaxysql_b200/_build/, which git ignores.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "_build")
SO = os.path.join(OUT, "libgsql_gpu.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SOURCES = ["ctx.cu", "join.cu", "agg.cu", "xchg.cu", "scan.cu", "serde.cu", "bloom.cu", "sort.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [
    *ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-Xptxas", "-v", "-DGSQL_BUILD",
]


def _stamp() -> str:
    h = hashlib.sha1()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT, exist_ok=True)
    stamp_file = os.path.join(OUT, "stamp")
    stamp = _stamp()
    if not force and os.path.exists(SO) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return SO
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]

    def compile_one(src):
        obj = os.path.join(OUT, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(os.path.join(OUT, src + ".log"), "w") as fh:
            fh.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [NVCC, "-shared", "-o", SO, *objs, *ARCH, "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
