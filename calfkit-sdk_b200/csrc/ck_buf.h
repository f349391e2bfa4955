// Owning buffers of the handle (ck_api.cu): device memory (ck_buf) and page-locked host memory (ck_pinned).  Host code
// only; kernels take the raw pointer .p.  A buffer is either empty (p null, cap 0) or holds cap elements it owns: a
// failed allocation empties it, so it never holds a freed pointer or claims room it does not have.
#pragma once
#include <cstddef>

#include <cuda_runtime_api.h>

template <class T, bool Pinned>
struct ck_buffer {
    T* p = nullptr;
    size_t cap = 0;                                    // elements

    ck_buffer() = default;
    ck_buffer(const ck_buffer&) = delete;
    ck_buffer& operator=(const ck_buffer&) = delete;
    ck_buffer(ck_buffer&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ck_buffer& operator=(ck_buffer&& o) noexcept {
        if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    ~ck_buffer() { release(); }

    // room for at least n elements.  Returns at once when there is.  Otherwise waits for `s` (work queued there may still
    // read the buffer; a failed wait returns its error and leaves the buffer as it was), frees the buffer, then allocates
    // one of exactly n elements: old and new never hold memory at the same time.  keep > 0 copies the first `keep`
    // elements (at most cap) over, so there the new buffer is allocated before the old one is freed.  A failed allocation
    // or copy leaves the buffer empty and returns the error
    cudaError_t reserve(size_t n, cudaStream_t s, size_t keep = 0) {
        if (n <= cap) return cudaSuccess;
        if (p) { cudaError_t e = cudaStreamSynchronize(s); if (e != cudaSuccess) return e; }
        if (keep > cap) keep = cap;
        if (!keep) release();
        T* q = nullptr;
        cudaError_t e = Pinned ? cudaMallocHost((void**)&q, sizeof(T) * n) : cudaMalloc((void**)&q, sizeof(T) * n);
        if (e == cudaSuccess && keep && (e = cudaMemcpy(q, p, sizeof(T) * keep, cudaMemcpyDefault)) != cudaSuccess) free_(q);
        release();
        if (e != cudaSuccess) return e;
        p = q; cap = n;
        return cudaSuccess;
    }

    void release() { if (p) free_(p); p = nullptr; cap = 0; }

private:
    static void free_(T* q) { if (Pinned) cudaFreeHost(q); else cudaFree(q); }
};

template <class T> using ck_buf = ck_buffer<T, false>;
template <class T> using ck_pinned = ck_buffer<T, true>;
