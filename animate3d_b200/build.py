"""Build liba3d.so (sm_90a only) in-tree with nvcc.  `python -m animate3d_b200.build [--force]`.

The .so and the object files are build products (git-ignored); the package loads the library from next to this file."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "liba3d.so")
OBJ = os.path.join(HERE, "build")
SOURCES = ["a3d_api.cu", "a3d_gemm.cu", "a3d_attn.cu", "a3d_ops.cu", "a3d_raster.cu", "a3d_raster_pre.cu", "a3d_deform.cu", "a3d_arap.cu",
           "a3d_mesh.cu", "a3d_clip.cu"]
# index-defining rasterizer arithmetic must not be contracted into FMAs (bit parity with oracle/raster_oracle.py)
EXTRA = {"a3d_raster_pre.cu": ["--fmad=false"]}
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for fn in sorted(os.listdir(root)):
            with open(os.path.join(root, fn), "rb") as f:
                h.update(fn.encode())
                h.update(f.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "digest.txt")
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; liba3d.so cannot be built (and there is no fallback path)")

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, *EXTRA.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, *ARCH],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
