// TEST INFRASTRUCTURE ONLY: the handle's owning buffers (csrc/ck_buf.h) built with g++ against the CUDA runtime, on their own
//   buf_host fail   no usable device: every reserve fails and leaves the buffer empty; moves and destructors stay safe
//   buf_host grow   a device: reserve grows, a reserve that fits changes nothing, keep carries the prefix over
// Prints one line per failed check and exits 1 if there was any.  Not covered: a failed reserve on a buffer that holds
// memory, which needs an allocation to fail on a device (without exhausting a shared GPU's memory there is no way to).
#include <cstdio>
#include <cstring>
#include <utility>

#include "ck_buf.h"

static int failures = 0;
#define CHECK(c) do { if (!(c)) { printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); failures++; } } while (0)

template <class B> static void fail_case() {
    B b;
    cudaError_t e = b.reserve(1000, nullptr);
    CHECK(e != cudaSuccess);
    CHECK(b.p == nullptr && b.cap == 0);
    CHECK(b.reserve(1000, nullptr, 10) == e);          // fails the same way again, with or without a prefix to keep
    CHECK(b.p == nullptr && b.cap == 0);
    CHECK(b.reserve(0, nullptr) == cudaSuccess);       // no room asked for: no call
    B moved(std::move(b));
    CHECK(moved.p == nullptr && moved.cap == 0 && b.p == nullptr && b.cap == 0);
    B assigned;
    assigned = std::move(moved);
    CHECK(assigned.p == nullptr && assigned.cap == 0 && moved.p == nullptr);
    printf("reserve failed with %s\n", cudaGetErrorName(e));
}   // the empty and moved-from buffers are destroyed here

template <class B> static void grow_case(cudaStream_t s) {
    int src[100], back[100];
    for (int i = 0; i < 100; i++) src[i] = 7 * i + 1;
    B b;
    CHECK(b.reserve(100, s) == cudaSuccess);
    CHECK(b.p != nullptr && b.cap == 100);
    int* p0 = b.p;
    CHECK(cudaMemcpy(b.p, src, sizeof src, cudaMemcpyDefault) == cudaSuccess);
    CHECK(b.reserve(60, s) == cudaSuccess && b.reserve(100, s) == cudaSuccess);
    CHECK(b.p == p0 && b.cap == 100);                  // it fits: the same buffer
    CHECK(b.reserve(1000, s, 100) == cudaSuccess);
    CHECK(b.cap == 1000);
    memset(back, 0, sizeof back);
    CHECK(cudaMemcpy(back, b.p, sizeof back, cudaMemcpyDefault) == cudaSuccess);
    CHECK(memcmp(back, src, sizeof src) == 0);         // the kept prefix
    CHECK(cudaMemcpy(b.p + 100, src, sizeof src, cudaMemcpyDefault) == cudaSuccess);
    CHECK(b.reserve(2000, s, 1 << 20) == cudaSuccess);   // keep beyond cap: the whole old buffer
    CHECK(b.cap == 2000);
    memset(back, 0, sizeof back);
    CHECK(cudaMemcpy(back, b.p + 100, sizeof back, cudaMemcpyDefault) == cudaSuccess);
    CHECK(memcmp(back, src, sizeof src) == 0);
    CHECK(b.reserve(5000, s) == cudaSuccess);
    CHECK(b.cap == 5000);
    int* p1 = b.p;
    B moved(std::move(b));
    CHECK(moved.p == p1 && moved.cap == 5000 && b.p == nullptr && b.cap == 0);
    B assigned;
    CHECK(assigned.reserve(10, s) == cudaSuccess);     // freed by the assignment below
    assigned = std::move(moved);
    CHECK(assigned.p == p1 && assigned.cap == 5000 && moved.p == nullptr && moved.cap == 0);
    assigned.release();
    CHECK(assigned.p == nullptr && assigned.cap == 0);
    CHECK(assigned.reserve(20, s) == cudaSuccess && assigned.cap == 20);
}

int main(int argc, char** argv) {
    if (argc != 2) { printf("usage: buf_host fail|grow\n"); return 2; }
    if (!strcmp(argv[1], "fail")) {
        fail_case<ck_buf<int>>();
        fail_case<ck_pinned<int>>();
    } else if (!strcmp(argv[1], "grow")) {
        cudaStream_t s = nullptr;
        CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess);
        grow_case<ck_buf<int>>(s);
        grow_case<ck_pinned<int>>(s);
        CHECK(cudaStreamDestroy(s) == cudaSuccess);
        CHECK(cudaGetLastError() == cudaSuccess);      // no free of a pointer the runtime does not know
    } else {
        printf("usage: buf_host fail|grow\n"); return 2;
    }
    if (!failures) printf("ok\n");
    return failures ? 1 : 0;
}
