// TEST INFRASTRUCTURE ONLY.  The shipped snappy decoder (csrc/ck_snappy.cuh) compiled by g++ as one lane, so that the CPU
// suite holds it against Google snappy (tests/test_snappy_hostsim.py).  Nothing in the product links or loads this file.
#include "ck_snappy.cuh"

// the walk of the section z[0, zn) as the host lists its chunks: blocks (their input offset, input length and declared
// length in t[3 i .. 3 i + 2], at most cap of them), or -1 when the section cannot be walked
extern "C" long long sn_host_walk(const u8* z, unsigned long long zn, unsigned long long* t, u32 cap) {
    ck_sn_walker w;
    ck_sn_begin(z, zn, w);
    unsigned long long off; u32 len, dl;
    long long k = 0;
    int r;
    while ((r = ck_sn_next(z, zn, w, &off, &len, &dl)) > 0) {
        if ((u32)k >= cap) return -1;
        t[3 * k] = off; t[3 * k + 1] = len; t[3 * k + 2] = dl;
        k++;
    }
    return r < 0 ? -1 : k;
}

// the raw block z[0, zn) decoded into out[0, cap) as ck_rb_snappy_kernel decodes it: decoded length, or -1
extern "C" long long sn_host_decode(const u8* z, u32 zn, u8* out, u32 cap) {
    return ck_sn_decode_block(z, zn, out, cap, 0);
}

// the decoded length of the raw block z[0, zn) as the walk and the decoder read it: 1 and *len, or 0 when refused
extern "C" int sn_host_varint(const u8* z, u32 zn, u32* len) {
    u32 ip;
    return ck_sn_varint(z, zn, &ip, len) ? 1 : 0;
}
