"""Build libfocoos_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m focoos_b200.csrc.build [--force]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SOURCES = ["conv_simt.cu", "conv_tc.cu", "pool_resize.cu", "norm_attn.cu", "msda.cu", "select.cu", "head_fused.cu", "mf_ops.cu", "bisenet_ops.cu", "criterion.cu", "optim.cu", "bwd_conv_norm.cu", "bwd_attn.cu", "wgrad_tc.cu", "mask_png.cu", "sem_seg.cu", "box_ap.cu"]
HEADERS = ["common.cuh", "tma.cuh", "wgmma.cuh", os.path.join(ROOT, "include", "focoos_b200.h")]
LIB_DIR = os.path.join(os.path.dirname(HERE), "lib")
LIB = os.path.join(LIB_DIR, "libfocoos_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-I", os.path.join(ROOT, "include"), "-I", HERE]


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        p = f if os.path.isabs(f) else os.path.join(HERE, f)
        with open(p, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    stamp = os.path.join(LIB_DIR, "build.sha256")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(HERE, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose and out:
            print(out)
    link = [NVCC, "-shared", "-o", LIB, *objs, *ARCH, "-lcudart"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
