"""TEST INFRASTRUCTURE ONLY: Google snappy as pyarrow bundles it, the reference the device snappy decoder is held against.

  compress(data)    one raw snappy block (snappy::RawCompress through pyarrow.compress)
  decompress(z)     snappy's verdict on z as one raw block (snappy::GetUncompressedLength, then RawUncompress through
                    pyarrow.decompress): its bytes, or None

pyarrow returns its output buffer untrimmed, so decompress() passes the block's own varint as the decompressed size: with
a larger size the bytes behind the output would be uninitialised.  A varint that the plain reading below does not take
(cut off, longer than 5 bytes) is passed as size 0, so that snappy's own varint check gives the verdict.  A block that
declares more than 64 MiB and more than 22 times its own size is refused without a call: no element emits more than 64/3
bytes per input byte, so snappy refuses it too, and allocating the declared size is not worth it.  available() is False
without pyarrow; tests that need it at test time skip then (`need()`)."""
import pytest

RATIO = 22


def available() -> bool:
    try:
        import pyarrow  # noqa: F401
    except ImportError:
        return False
    return True


def need():
    """pyarrow, or skip the calling test"""
    if not available():
        pytest.skip("pyarrow (snappy) not installed")
    import pyarrow
    return pyarrow


def version() -> str:
    return need().__version__


def compress(data: bytes) -> bytes:
    return need().compress(bytes(data), codec="snappy", asbytes=True)


def declared(z: bytes):
    """the varint at the start of z read plainly (at most 5 bytes, no range check), or None when it is cut off or longer"""
    v = 0
    for k in range(min(5, len(z))):
        v |= (z[k] & 0x7F) << (7 * k)
        if z[k] < 0x80:
            return v
    return None


def decompress(z: bytes):
    pa = need()
    n = declared(z)
    if n is not None and n > (64 << 20) and n > RATIO * len(z):
        return None
    try:
        out = pa.decompress(bytes(z), decompressed_size=n if n is not None and n < (1 << 32) else 0, codec="snappy", asbytes=True)
    except OSError:
        return None
    except pa.ArrowInvalid as e:            # the output was smaller than snappy's own reading of the varint
        raise AssertionError(f"snappy read a varint the plain reading did not: {e}") from e
    return bytes(out)
