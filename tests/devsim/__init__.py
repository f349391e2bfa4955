"""TEST INFRASTRUCTURE ONLY: nvcc build of launchers that run the shipped emitter, scan and key-hash device code on
inputs a test makes (tests/test_gpu_kernels.py)."""
import ctypes
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "calfkit-sdk_b200", "csrc")
_LIB = os.path.join(HERE, "libck_devsim.so")


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, "devsim.cu"), os.path.abspath(__file__)] + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + \
        [os.path.join(CSRC, "ck_common.h")]
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "-Xcompiler", "-fPIC,-Wno-stringop-overflow", "-shared", "-I", CSRC, "-o", _LIB, srcs[0]])
    return _LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        p, u32, i64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_longlong
        _lib.ck_dev_emit.argtypes = [p, p, u32, p, p, p, p, p, u32, p, i64]
        _lib.ck_dev_scan.argtypes = [p, u32, p, u32, p, p]
        _lib.ck_dev_murmur2_key.argtypes = [ctypes.c_int, p, p, u32, p, u32, p, p]
        for f in (_lib.ck_dev_emit, _lib.ck_dev_scan, _lib.ck_dev_murmur2_key):
            f.restype = ctypes.c_int
    return _lib


def check(err: int) -> None:
    if err:
        raise RuntimeError(f"devsim launch failed: cudaError {err}")
