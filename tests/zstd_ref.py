"""TEST INFRASTRUCTURE ONLY: libzstd (libzstd.so.1) through ctypes, the reference the device zstd decoder is held against.

  compress(data, ...)   one frame from ZSTD_compress2 with the parameters set by ZSTD_CCtx_setParameter: level,
                        windowLog, strategy, checksumFlag, contentSizeFlag, long-distance matching, targetCBlockSize
  stream(data, ...)     one frame from ZSTD_compressStream2 fed in pieces, with or without a flush after each: no
                        Frame_Content_Size, a window descriptor
  decompress(z)         the verdict of a DCtx with default parameters on the section z as one frame: its bytes, or None

decompress() runs ZSTD_decompressStream, the decoder that applies the DCtx's parameters (windowLogMax 27, the block
maximum); the input's first byte goes in a call of its own, so that libzstd never takes its single-pass shortcut (which
skips both).  Like the device, it refuses a section that is not exactly one zstd frame: a skippable frame, a second frame
or any byte after the frame.  lib() is None when libzstd.so.1 cannot be loaded; tests that compress at test time skip
then (`need()`)."""
import ctypes as C

import pytest

MAGIC = b"\x28\xb5\x2f\xfd"
C_LEVEL, C_WLOG, C_STRATEGY, C_LDM = 100, 101, 107, 160
C_CONTENT_SIZE, C_CHECKSUM = 200, 201
C_TARGET_CBLOCK = 1003                  # ZSTD_c_targetCBlockSize (ZSTD_c_experimentalParam6)
E_CONTINUE, E_FLUSH, E_END = 0, 1, 2

_lib = []


class _Buf(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def lib():
    if not _lib:
        try:
            L = C.CDLL("libzstd.so.1")
        except OSError:
            _lib.append(None)
            return None
        L.ZSTD_versionString.restype = C.c_char_p
        L.ZSTD_createCCtx.restype = C.c_void_p
        L.ZSTD_createDCtx.restype = C.c_void_p
        L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        L.ZSTD_freeDCtx.argtypes = [C.c_void_p]
        L.ZSTD_isError.argtypes = [C.c_size_t]
        L.ZSTD_getErrorName.argtypes = [C.c_size_t]
        L.ZSTD_getErrorName.restype = C.c_char_p
        L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ZSTD_CCtx_setParameter.restype = C.c_size_t
        L.ZSTD_compressBound.argtypes = [C.c_size_t]
        L.ZSTD_compressBound.restype = C.c_size_t
        L.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.ZSTD_compress2.restype = C.c_size_t
        L.ZSTD_compressStream2.argtypes = [C.c_void_p, C.POINTER(_Buf), C.POINTER(_Buf), C.c_int]
        L.ZSTD_compressStream2.restype = C.c_size_t
        L.ZSTD_decompressStream.argtypes = [C.c_void_p, C.POINTER(_Buf), C.POINTER(_Buf)]
        L.ZSTD_decompressStream.restype = C.c_size_t
        _lib.append(L)
    return _lib[0]


def need():
    """the library, or skip the calling test"""
    L = lib()
    if L is None:
        pytest.skip("libzstd.so.1 not found")
    return L


def version() -> str:
    return need().ZSTD_versionString().decode()


def _cctx(level=3, window_log=0, strategy=0, checksum=False, content_size=True, ldm=False, target_cblock=0):
    L = need()
    cc = L.ZSTD_createCCtx()
    for p, v in ((C_LEVEL, level), (C_WLOG, window_log), (C_STRATEGY, strategy), (C_CHECKSUM, int(checksum)),
                 (C_CONTENT_SIZE, int(content_size)), (C_LDM, 1 if ldm else 0), (C_TARGET_CBLOCK, target_cblock)):
        r = L.ZSTD_CCtx_setParameter(cc, p, v)
        assert not L.ZSTD_isError(r), (p, v, L.ZSTD_getErrorName(r))
    return cc


def compress(data: bytes, **kw) -> bytes:
    """one frame of `data` (ZSTD_compress2); kw: level, window_log, strategy, checksum, content_size, ldm, target_cblock"""
    L = need()
    cc = _cctx(**kw)
    try:
        cap = L.ZSTD_compressBound(len(data))
        out = C.create_string_buffer(cap)
        r = L.ZSTD_compress2(cc, out, cap, bytes(data), len(data))
        assert not L.ZSTD_isError(r), L.ZSTD_getErrorName(r)
        return out.raw[:r]
    finally:
        L.ZSTD_freeCCtx(cc)


def stream(data: bytes, piece: int = 4096, flush: bool = False, **kw) -> bytes:
    """one frame of `data` fed to ZSTD_compressStream2 `piece` bytes at a time (flushing after each when `flush`): the
    streaming shape, with no Frame_Content_Size"""
    L = need()
    cc = _cctx(**kw)
    try:
        cap = L.ZSTD_compressBound(len(data)) + 1024 + 16 * (len(data) // max(piece, 1) + 1)
        out = C.create_string_buffer(cap)
        src = C.create_string_buffer(bytes(data), max(len(data), 1))
        ob = _Buf(C.cast(out, C.c_void_p), cap, 0)
        for a in range(0, len(data), piece):
            ib = _Buf(C.cast(src, C.c_void_p).value + a, min(piece, len(data) - a), 0)
            while ib.pos < ib.size:
                r = L.ZSTD_compressStream2(cc, C.byref(ob), C.byref(ib), E_CONTINUE)
                assert not L.ZSTD_isError(r)
            if flush:
                e = _Buf(None, 0, 0)
                while L.ZSTD_compressStream2(cc, C.byref(ob), C.byref(e), E_FLUSH):
                    pass
        e = _Buf(None, 0, 0)
        while True:
            r = L.ZSTD_compressStream2(cc, C.byref(ob), C.byref(e), E_END)
            assert not L.ZSTD_isError(r)
            if r == 0:
                break
        return out.raw[:ob.pos]
    finally:
        L.ZSTD_freeCCtx(cc)


def decompress(z: bytes, cap: int = 8 << 20):
    """libzstd's verdict on the section z as exactly one zstd frame: its bytes, or None"""
    L = need()
    z = bytes(z)
    if z[:4] != MAGIC:
        return None                      # not a zstd frame (a skippable one included)
    dc = L.ZSTD_createDCtx()
    try:
        src = C.create_string_buffer(z, len(z))
        out = C.create_string_buffer(cap)
        ob = _Buf(C.cast(out, C.c_void_p), 0, 0)
        ib = _Buf(C.cast(src, C.c_void_p), 1, 0)
        r = L.ZSTD_decompressStream(dc, C.byref(ob), C.byref(ib))
        if L.ZSTD_isError(r):
            return None
        ob.size, ib.size = cap, len(z)
        for _ in range(64):
            before = (ib.pos, ob.pos)
            r = L.ZSTD_decompressStream(dc, C.byref(ob), C.byref(ib))
            if L.ZSTD_isError(r):
                return None
            if r == 0 or (ib.pos, ob.pos) == before:
                break
        if r != 0 or ib.pos != len(z):
            return None                  # the frame is not finished, or something follows it
        return out.raw[:ob.pos]
    finally:
        L.ZSTD_freeDCtx(dc)
