"""TEST INFRASTRUCTURE ONLY: builds of the shipped snappy decoder (csrc/ck_snappy.cuh) on its own.

  host_lib()  g++, one lane: raw blocks and whole sections on the CPU (tests/test_snappy_hostsim.py,
              tests/test_snappy_batches_golden.py)
  lib()       nvcc for sm_90a, a warp per block (tests/test_gpu_snappy.py)

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
        srcs = [os.path.join(HERE, src), os.path.join(CSRC, "ck_snappy.cuh")]
        key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"ck_snappy_{kind}_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(cmd + ["-I", CSRC, "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        _libs[kind] = ctypes.CDLL(so)
    return _libs[kind]


def host_lib() -> ctypes.CDLL:
    L = _build("host", "snappydec_host.cpp", ["g++", "-O2", "-std=c++17", "-shared", "-fPIC"])
    p, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
    L.sn_host_walk.argtypes = [p, u64, p, u32]
    L.sn_host_walk.restype = ctypes.c_longlong
    L.sn_host_decode.argtypes = [p, u32, p, u32]
    L.sn_host_decode.restype = ctypes.c_longlong
    L.sn_host_varint.argtypes = [p, u32, p]
    L.sn_host_varint.restype = ctypes.c_int
    return L


def lib() -> ctypes.CDLL:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    L = _build("dev", "snappydec.cu", [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"])
    p = ctypes.c_void_p
    L.snappy_blocks.argtypes = [p, p, ctypes.c_uint32, p, p, p]
    L.snappy_blocks.restype = ctypes.c_int
    return L


def _buf(b: bytes):
    return ctypes.create_string_buffer(bytes(b) + b"\0" * 64, len(b) + 64)


def walk(sec: bytes):
    """the host's walk of a records section: [(input offset, input length, declared length)], or None when refused"""
    cap = len(sec) // 5 + 2
    t = (ctypes.c_uint64 * (3 * cap))()
    n = host_lib().sn_host_walk(_buf(sec), len(sec), t, cap)
    return None if n < 0 else [(t[3 * i], t[3 * i + 1], t[3 * i + 2]) for i in range(n)]


def declared(z: bytes):
    """the raw block's declared length as the host build reads its varint, or None"""
    n = ctypes.c_uint32(0)
    return n.value if host_lib().sn_host_varint(_buf(z), len(z), ctypes.byref(n)) else None


def decode_block(z: bytes, cap: int | None = None):
    """the host build on the raw block z decoded into cap bytes (default: its declared length, 0 when unreadable): the
    decoded bytes, or None when refused"""
    if cap is None:
        cap = declared(z) or 0
    out = ctypes.create_string_buffer(cap + 64)
    r = host_lib().sn_host_decode(_buf(z), len(z), out, cap)
    return None if r < 0 else out.raw[:r]


def decode_section(sec: bytes):
    """a records section as the device decodes it: walked, then every block into its place; bytes or None"""
    w = walk(sec)
    if w is None:
        return None
    out = bytearray()
    for off, ln, dl in w:
        d = decode_block(sec[off:off + ln], dl)
        if d is None:
            return None
        out += d
    return bytes(out)
