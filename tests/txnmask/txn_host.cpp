// TEST INFRASTRUCTURE ONLY: the transaction rule (csrc/ck_txn.h) built with g++ on its own
#include "ck_txn.h"

extern "C" uint32_t txn_crc32c(const uint8_t* p, uint64_t n) { return ck_txn_crc32c(p, n); }

extern "C" long long txn_mask(const uint8_t* buf, uint64_t n, const uint64_t* run_start, uint32_t nruns, const uint32_t* abort_run,
                              const int64_t* abort_pid, const int64_t* abort_first, uint32_t naborts, uint8_t* mask, uint64_t cap) {
    return ck_txn_mask(buf, n, run_start, nruns, abort_run, abort_pid, abort_first, naborts, mask, cap);
}

// what a batch comes out as on the device, per complete batch: the flag ck_submit_recordbatch gives it (control batches
// their own verdict, the others the mask's; mask NULL: read_uncommitted) where it passes the device's framing check, else bad
extern "C" long long txn_verdicts(const uint8_t* buf, uint64_t n, const uint8_t* mask, uint8_t* out, uint64_t cap) {
    uint64_t pos = 0, end;
    long long b = 0;
    for (; (end = ck_txn_frame_end(buf, n, pos)) != 0 && (uint64_t)b < cap; pos = end, b++) {
        const uint8_t* f = buf + pos;
        int type;
        int flag = (f[22] & CK_TXN_CONTROL) ? ck_txn_control(f, end - pos, &type) : mask && mask[b] ? CK_TXN_HIDE : CK_TXN_SHOW;
        out[b] = ck_txn_framed(f, end - pos, true) ? (uint8_t)flag : (uint8_t)CK_TXN_BAD;
    }
    return b;
}
