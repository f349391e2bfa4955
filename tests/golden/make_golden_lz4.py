"""Writes tests/golden/lz4_frames.json: seeded inputs and the LZ4 frames the system liblz4 (LZ4F_compressFrame) makes of
them, with every frame flag (linked blocks, block checksum, content checksum, content size), block sizes of 64 KB to
4 MB, compressible and incompressible data, and XXH32 vectors (read from the content checksums liblz4 writes).
The inputs are not stored: `inputs()` makes them again from their seeds (tests/test_lz4_oracle.py imports it); the frames
are stored as liblz4 wrote them (base64).

    python tests/golden/make_golden_lz4.py        (needs liblz4; the tests only read the JSON)
"""
import base64
import ctypes
import ctypes.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "..", "calfkit-sdk_b200"), os.path.join(HERE, "..", "..")]


class FrameInfo(ctypes.Structure):
    _fields_ = [("blockSizeID", ctypes.c_int), ("blockMode", ctypes.c_int), ("contentChecksumFlag", ctypes.c_int),
                ("frameType", ctypes.c_int), ("contentSize", ctypes.c_ulonglong), ("dictID", ctypes.c_uint),
                ("blockChecksumFlag", ctypes.c_int)]


class Prefs(ctypes.Structure):
    _fields_ = [("frameInfo", FrameInfo), ("compressionLevel", ctypes.c_int), ("autoFlush", ctypes.c_uint),
                ("favorDecSpeed", ctypes.c_uint), ("reserved", ctypes.c_uint * 3)]


def lib():
    L = ctypes.CDLL(ctypes.util.find_library("lz4") or "liblz4.so.1")
    L.LZ4F_compressFrameBound.restype = ctypes.c_size_t
    L.LZ4F_compressFrameBound.argtypes = [ctypes.c_size_t, ctypes.c_void_p]
    L.LZ4F_compressFrame.restype = ctypes.c_size_t
    L.LZ4F_compressFrame.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p]
    L.LZ4F_isError.argtypes = [ctypes.c_size_t]
    L.LZ4_versionString.restype = ctypes.c_char_p
    return L


def compress(L, data: bytes, block_id=0, linked=False, block_sum=False, content_sum=False, content_size=False, level=0,
             default=False):
    """default: liblz4's default preferences (NULL), which link the blocks of a frame of more than one block"""
    p = Prefs()
    p.frameInfo.blockSizeID, p.frameInfo.blockMode = block_id, 0 if linked else 1
    p.frameInfo.contentChecksumFlag, p.frameInfo.blockChecksumFlag = int(content_sum), int(block_sum)
    p.frameInfo.contentSize = len(data) if content_size else 0
    p.compressionLevel = level
    pp = None if default else ctypes.byref(p)
    cap = L.LZ4F_compressFrameBound(len(data), pp)
    out = ctypes.create_string_buffer(cap)
    n = L.LZ4F_compressFrame(out, cap, data, len(data), pp)
    assert not L.LZ4F_isError(n), n
    return out.raw[:n]


def inputs():
    from calfkit import synth
    from oracle import kafka_batch as kb
    rng = np.random.default_rng(20261016)
    recs = synth.tool_events(80, seed=111)
    records = b""                                # the records section of a batch of the first records (up to 20 KB)
    for i, r in enumerate(recs):
        rec = kb.encode_record(kb.calfkit_record(r, f"corr-{i:06d}"), i, 0)
        if len(records) + len(rec) > 20_000:
            break
        records += rec
    return {
        "empty": b"",
        "one_byte": b"x",
        "twelve": b"abcdefghijkl",
        "thirteen": b"aaaaaaaaaaaaa",
        "records_20k": records,
        "one_byte_run_100k": b"\x07" * 100_000,
        "random_3k": rng.integers(0, 256, 3000, dtype=np.uint8).tobytes(),
        "period_251": bytes(range(251)) * 300,
        "period_251_1500k": bytes(range(251)) * 6000,     # liblz4 lowers the block size to fit the input: larger inputs
    }


def main():
    L = lib()
    data = inputs()
    common = [k for k in data if k not in ("random_3k", "period_251_1500k")]
    variants = [
        ("default", {"default": True}, common),
        ("independent", {}, ["records_20k", "random_3k", "period_251"]),
        ("linked", {"linked": True}, ["records_20k", "period_251"]),
        ("block_checksum", {"block_sum": True}, ["records_20k", "random_3k", "one_byte"]),
        ("content_checksum", {"content_sum": True}, common),
        ("content_size", {"content_size": True}, ["records_20k", "empty"]),
        ("all_flags", {"linked": True, "block_sum": True, "content_sum": True, "content_size": True}, ["records_20k", "period_251"]),
        ("block_256k", {"block_id": 5}, ["period_251_1500k"]),
        ("block_1m", {"block_id": 6, "content_sum": True}, ["period_251_1500k"]),
        ("block_4m", {"block_id": 7}, ["period_251_1500k"]),
        ("hc_level_9", {"level": 9}, ["records_20k", "one_byte_run_100k"]),
    ]
    frames = [{"variant": v, "input": name, "frame": base64.b64encode(compress(L, data[name], **kw)).decode()}
              for v, kw, names in variants for name in names]
    # XXH32: liblz4's content checksum of each input is xxh32(input, seed 0)
    xxh = []
    for name, d in data.items():
        f = compress(L, d, content_sum=True)
        xxh.append({"input": name, "xxh32": int.from_bytes(f[-4:], "little")})
    out = {"liblz4": L.LZ4_versionString().decode(), "frames": frames, "xxh32": xxh}
    with open(os.path.join(HERE, "lz4_frames.json"), "w") as fh:
        json.dump(out, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
