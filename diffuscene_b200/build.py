"""Build libdiffuscene_b200.so in-tree with nvcc for sm_90a (no JIT cache, no torch extension).

    python -m diffuscene_b200.build          # or diffuscene_b200.build.build()

The shared library exports only the C ABI of include/diffuscene_b200.h; Python binds it with ctypes
(diffuscene_b200/capi.py).  nvcc cross-compiles without a GPU, so this also runs on CPU-only boxes.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdiffuscene_b200.so")
SOURCES = ["engine.cu", "plan.cpp", "pointwise.cu", "gemm_simt.cu", "gemm_tc.cu", "gemm_ln.cu", "gemm_attn.cu", "backward.cu", "train.cu", "room_encoder.cu", "shape_ae.cu", "text_encoder.cu", "scene_eval.cu", "vgg16.cu", "manifold.cu", "inception.cu", "fid_stats.cu", "render.cu", "resize.cu", "scene_batch.cu"]
HEADERS = ["common.cuh", "kernels.cuh", "tc_common.cuh", "placement.cuh", "plan.h", "engine_internal.h", os.path.join("..", "..", "include", "diffuscene_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    stamp = os.path.join(LIB_DIR, "build.sha256")
    digest = _digest()
    if not force and os.path.exists(LIB_PATH) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed on %s" % src)
        if verbose and out:
            print(out.decode())
    cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
