"""Builds libk210yolo_b200.so in-tree with nvcc for sm_90a (no torch extension machinery: the library is a
plain C-ABI .so with cudart linked statically, so it loads — and its symbols can be checked — on a box
without a GPU or libcuda)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libk210yolo_b200.so")
SOURCES = ["conv_simt.cu", "gemm_tc.cu", "detect.cu", "net.cu", "region_layer_abi.cu", "preprocess.cu", "jpeg.cu", "jpeg_progressive.cu", "png.cu", "jpeg_encode.cu", "render.cu", "evaluate.cu", "evaluate_mot.cu", "track.cu", "bytetrack.cu", "ocsort.cu", "comm.cu"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC", "-shared"]


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", f)
                                                                 for f in os.listdir(os.path.join(HERE, "..", "include"))]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("K2Y_NVCC_EXTRA", "").split()   # extra nvcc flags, for development builds only
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building libk210yolo_b200.so")
    if verbose:
        print(r.stdout)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
