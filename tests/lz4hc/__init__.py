"""TEST INFRASTRUCTURE ONLY: nvcc build of a launcher that runs the shipped hash-chain LZ4 block compressor
(ck_lz4_block_hc, csrc/ck_lz4.cuh) on blocks a test makes (tests/test_gpu_kafka_lz4_level.py).  The header stands alone,
so the build takes seconds; it goes to a temporary directory, keyed by the sources, and leaves the tree untouched."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "calfkit-sdk_b200", "csrc")
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(HERE, "lz4hc.cu"), os.path.join(CSRC, "ck_lz4.cuh")]
        key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"ck_lz4hc_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
            subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                                   "-shared", "-I", CSRC, "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        _lib = ctypes.CDLL(so)
        p = ctypes.c_void_p
        _lib.lz4hc_blocks.argtypes = [p, p, ctypes.c_uint32, p, p, p, ctypes.c_uint32]
        _lib.lz4hc_blocks.restype = ctypes.c_int
    return _lib
