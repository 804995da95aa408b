"""Build libmoco_b200.so in-tree with nvcc for sm_90a (no torch extension machinery:
the library is plain C ABI, loaded with ctypes)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmoco_b200.so")
SOURCES = ["capi.cu", "nce_support.cu", "nce_tail.cu", "nce_sweep_sm90.cu", "queue_shuffle.cu", "ema.cu", "bn_nhwc.cu",
           "pool_nhwc.cu", "conv1x1_sm90.cu", "knn_sm90.cu", "augment.cu"]
HEADERS = ["common.cuh", "bn_reduce.cuh", "sm90_ptx.cuh", "tc_common.cuh", "conv1x1_skeleton.cuh", "nce_rows.cuh",
           os.path.join("..", "..", "include", "moco_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared",
]


def _newer(a, b):
    return os.path.getmtime(a) > os.path.getmtime(b)


def needs_build():
    if not os.path.exists(LIB):
        return True
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(_newer(d, LIB) for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libmoco_b200.so")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
