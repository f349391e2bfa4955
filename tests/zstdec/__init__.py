"""TEST INFRASTRUCTURE ONLY: builds of the shipped zstd decoder (csrc/ck_zstd.cuh) on its own.

  host_lib()  g++, one lane: whole frames on the CPU (tests/test_zstd_hostsim.py, tests/test_zstd_batches_golden.py)
  lib()       nvcc for sm_90a, a warp per frame (tests/test_gpu_zstd.py)

The header stands alone, so each build takes seconds; it goes to a temporary directory, keyed by the sources, and leaves
the tree untouched."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "calfkit-sdk_b200", "csrc")
_libs = {}


def _build(kind: str, src: str, cmd) -> ctypes.CDLL:
    if kind not in _libs:
        srcs = [os.path.join(HERE, src), os.path.join(CSRC, "ck_zstd.cuh")]
        key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"ck_zstd_{kind}_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(cmd + ["-I", CSRC, "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        _libs[kind] = ctypes.CDLL(so)
    return _libs[kind]


def host_lib() -> ctypes.CDLL:
    L = _build("host", "zstdec_host.cpp", ["g++", "-O2", "-std=c++17", "-shared", "-fPIC"])
    p, u64 = ctypes.c_void_p, ctypes.c_uint64
    L.zs_host_bound.argtypes = [p, u64, p]
    L.zs_host_bound.restype = ctypes.c_int
    L.zs_host_decode.argtypes = [p, u64, p, u64]
    L.zs_host_decode.restype = ctypes.c_longlong
    return L


def lib() -> ctypes.CDLL:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    L = _build("dev", "zstdec.cu", [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"])
    p = ctypes.c_void_p
    L.zstd_frames.argtypes = [p, p, ctypes.c_uint32, p, p, p]
    L.zstd_frames.restype = ctypes.c_int
    return L


def _buf(b: bytes):
    return ctypes.create_string_buffer(bytes(b) + b"\0" * 64, len(b) + 64)


def bound(z: bytes):
    """the slot the host gives the frame z: its block walk's bound, or None when the header or the walk refuses it"""
    b = ctypes.c_uint64(0)
    return b.value if host_lib().zs_host_bound(_buf(z), len(z), ctypes.byref(b)) else None


def decode(z: bytes, cap: int | None = None):
    """the host build on the frame z, as the kernel decodes it into a slot of `cap` bytes (default: its bound, 0 when the
    host refuses it): the decoded bytes, or None when it is refused"""
    if cap is None:
        cap = bound(z) or 0
    out = ctypes.create_string_buffer(cap + 64)
    r = host_lib().zs_host_decode(_buf(z), len(z), out, cap)
    return None if r < 0 else out.raw[:r]
