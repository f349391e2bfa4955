"""Builds libcalfkit_b200.so in-tree for sm_90a (H100; nvcc cross-compiles without a GPU).

    python calfkit-sdk_b200/build.py [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libcalfkit_b200.so")
SRCS = [os.path.join(HERE, "csrc", "ck_api.cu")]
DEPS = SRCS + [os.path.join(HERE, "csrc", f) for f in ("ck_kernels.cuh", "ck_walk.cuh", "ck_float.cuh", "ck_canon.cuh", "ck_plan.cuh", "ck_gate.cuh", "ck_kafka.cuh", "ck_lz4.cuh", "ck_inflate.cuh", "ck_zstd.cuh", "ck_snappy.cuh", "ck_txn.h", "ck_buf.h", "ck_group.cuh", "ck_xsend.cuh", "ck_fanout2.cuh", "ck_walk_long.cuh", "ck_common.h")] + \
    [os.path.join(HERE, "..", "include", "calfkit_b200.h"), os.path.abspath(__file__)]   # this file: a changed nvcc command rebuilds


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in DEPS):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-Xcompiler", "-fPIC,-Wno-stringop-overflow", "-shared", "-o", LIB] + SRCS
    if verbose:
        cmd += ["-Xptxas", "-v"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose="--verbose" in sys.argv))
