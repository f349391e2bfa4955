"""TEST INFRASTRUCTURE ONLY: the transaction rule of the fetch path (csrc/ck_txn.h) built with g++ on its own.

  mask(buf, partitions)              ck_txn_mask: 1 for each batch read_committed skips as an aborted transaction's
  verdicts(buf, partitions, rc)      0 delivered / 1 bad / 2 skipped per complete batch, as the device ends up flagging it
  crc32c(data)                       the header's CRC32C, for writers of large batches

The header stands alone, so the build takes a second; it goes to a temporary directory, keyed by the sources, and leaves
the tree untouched."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "calfkit-sdk_b200", "csrc")
_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        srcs = [os.path.join(HERE, "txn_host.cpp"), os.path.join(CSRC, "ck_txn.h")]
        key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"ck_txn_host_{os.getuid()}_{key}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-I", CSRC, "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        p, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        L.txn_mask.argtypes = [p, u64, p, u32, p, p, p, u32, p, u64]
        L.txn_mask.restype = ctypes.c_longlong
        L.txn_verdicts.argtypes = [p, u64, p, p, u64]
        L.txn_verdicts.restype = ctypes.c_longlong
        L.txn_crc32c.argtypes = [p, u64]
        L.txn_crc32c.restype = ctypes.c_uint32
        _lib = L
    return _lib


def _arrays(partitions):
    starts = np.asarray([s for s, _ab in partitions], dtype=np.uint64)
    runs = np.asarray([r for r, (_s, ab) in enumerate(partitions) for _e in ab], dtype=np.uint32)
    pids = np.asarray([pid for _s, ab in partitions for pid, _f in ab], dtype=np.int64)
    firsts = np.asarray([f for _s, ab in partitions for _p, f in ab], dtype=np.int64)
    return starts, runs, pids, firsts


def crc32c(data: bytes) -> int:
    """CRC32C at native speed (oracle.kafka_batch.crc32c goes byte by byte in Python)"""
    return lib().txn_crc32c(data, len(data))


def mask(buf: bytes, partitions):
    """the mask, or None when the partitions are refused"""
    b = np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8)
    starts, runs, pids, firsts = _arrays(partitions)
    out = np.zeros(len(buf) // 61 + 1, dtype=np.uint8)
    nb = lib().txn_mask(b.ctypes.data, len(buf), starts.ctypes.data, len(starts), runs.ctypes.data, pids.ctypes.data,
                        firsts.ctypes.data, len(runs), out.ctypes.data, len(out))
    return None if nb < 0 else out[:nb]


def verdicts(buf: bytes, partitions, read_committed: bool) -> list[int]:
    m = mask(buf, partitions) if read_committed else None
    b = np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8)
    out = np.zeros(len(buf) // 61 + 1, dtype=np.uint8)
    nb = lib().txn_verdicts(b.ctypes.data, len(buf), None if m is None else m.ctypes.data, out.ctypes.data, len(out))
    return [int(x) for x in out[:nb]]
