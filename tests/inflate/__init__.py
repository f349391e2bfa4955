"""TEST INFRASTRUCTURE ONLY: builds of the shipped inflate core (csrc/ck_inflate.cuh) on its own.

  host_lib()  g++, one lane: raw deflate streams and whole gzip members on the CPU (tests/test_inflate_hostsim.py)
  lib()       nvcc for sm_90a, a warp per stream (tests/test_gpu_inflate.py)

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
        srcs = [os.path.join(HERE, src), os.path.join(CSRC, "ck_inflate.cuh")]
        key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"ck_inflate_{kind}_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(cmd + ["-I", CSRC, "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        _libs[kind] = ctypes.CDLL(so)
    return _libs[kind]


def host_lib() -> ctypes.CDLL:
    L = _build("host", "inflate_host.cpp", ["g++", "-O2", "-std=c++17", "-shared", "-fPIC"])
    p, u64 = ctypes.c_void_p, ctypes.c_uint64
    L.gz_host_inflate.argtypes = [p, u64, p, u64, p]
    L.gz_host_inflate.restype = ctypes.c_longlong
    L.gz_host_member.argtypes = [p, u64, p, u64, p]
    L.gz_host_member.restype = ctypes.c_longlong
    return L


def lib() -> ctypes.CDLL:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    L = _build("dev", "inflate.cu", [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"])
    p = ctypes.c_void_p
    L.inflate_streams.argtypes = [p, p, ctypes.c_uint32, p, p, p, p]
    L.inflate_streams.restype = ctypes.c_int
    L.inflate_members.argtypes = [p, p, ctypes.c_uint32, p, p, p]
    L.inflate_members.restype = ctypes.c_int
    return L


def _buf(b: bytes):
    return ctypes.create_string_buffer(bytes(b) + b"\0" * 64, len(b) + 64)


def inflate(stream: bytes, cap: int):
    """the host build on a raw deflate stream: (inflated bytes or None, bytes the stream took)"""
    out = ctypes.create_string_buffer(cap + 64)
    used = ctypes.c_uint64(0)
    r = host_lib().gz_host_inflate(_buf(stream), len(stream), out, cap, ctypes.byref(used))
    return (None if r < 0 else out.raw[:r]), used.value


def member(z: bytes):
    """the host build on a gzip member, as the kernel decodes it: its inflated bytes, or None when it is refused"""
    isize = ctypes.c_longlong(0)
    cap = min(int.from_bytes(z[-4:], "little"), 1 << 28) if len(z) >= 4 else 0
    out = ctypes.create_string_buffer(cap + 64)
    r = host_lib().gz_host_member(_buf(z), len(z), out, cap, ctypes.byref(isize))
    return None if r < 0 else out.raw[:r]
