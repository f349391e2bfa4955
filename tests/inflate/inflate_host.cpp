// TEST INFRASTRUCTURE ONLY.  The shipped inflate core (csrc/ck_inflate.cuh) compiled by g++ as one lane, so that the CPU
// suite holds it against zlib (tests/test_inflate_hostsim.py).  Nothing in the product links or loads this file.
#include <vector>
#include "ck_inflate.cuh"

// the raw deflate stream src[0, n) into out[0, cap): inflated length or -1; *used = bytes the stream took
extern "C" long long gz_host_inflate(const u8* src, unsigned long long n, u8* out, unsigned long long cap, unsigned long long* used) {
    static ck_gz_ws ws;
    *used = 0;
    return ck_inflate(src, n, out, cap, ws, 0, used);
}

// the gzip member z[0, zn) as ck_rb_gzip_kernel decodes it, the trailer's CRC32 included (here bit by bit): the header's
// ISIZE sizes the output; *isize = it (or -1 when the header is refused).  Returns the inflated length or -1
extern "C" long long gz_host_member(const u8* z, unsigned long long zn, u8* out, unsigned long long cap, long long* isize) {
    static ck_gz_ws ws;
    u32 hdr, sz;
    *isize = -1;
    if (!ck_gz_member(z, zn, &hdr, &sz)) return -1;
    *isize = sz;
    if (sz > cap) return -1;
    long long r = ck_gz_decode(z, zn, out, sz, ws, 0);
    if (r < 0 || ck_gz_crc32_bytes(out, (unsigned long long)r) != ck_gz_le32(z + zn - 8)) return -1;
    return r;
}
