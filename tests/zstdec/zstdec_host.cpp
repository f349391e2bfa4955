// TEST INFRASTRUCTURE ONLY.  The shipped zstd decoder (csrc/ck_zstd.cuh) compiled by g++ as one lane, so that the CPU
// suite holds it against libzstd (tests/test_zstd_hostsim.py).  Nothing in the product links or loads this file.
#include "ck_zstd.cuh"

// the frame z[0, zn) as the host sizes its slot: 1 and *bound = the block walk's bound, or 0 when the header or the walk
// refuses it
extern "C" int zs_host_bound(const u8* z, unsigned long long zn, unsigned long long* bound) {
    ck_zs_frame f;
    *bound = 0;
    return ck_zs_header(z, zn, f) && ck_zs_walk(z, zn, f, bound) ? 1 : 0;
}

// the frame z[0, zn) decoded into out[0, cap) as ck_rb_zstd_kernel decodes it: decoded length, or -1
extern "C" long long zs_host_decode(const u8* z, unsigned long long zn, u8* out, unsigned long long cap) {
    static ck_zs_ws ws;
    return ck_zs_decode(z, zn, out, cap, ws, 0);
}
