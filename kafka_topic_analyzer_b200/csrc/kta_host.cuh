// kta_host.cuh — host utilities of the library's host code (kta_api.cu, kta_logscan.cuh): the error text of the last failed
// call (fail, CU) and typed owners of device and pinned memory (DevBuf, PinnedBuf).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <utility>

#include "../../include/kta.h"

// the text kta_last_error returns, per thread
static thread_local char g_err[512] = "";

static int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(e_ == cudaErrorMemoryAllocation ? KTA_ERR_NOMEM : KTA_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                        cudaGetErrorString(e_), __FILE__, __LINE__);                                 \
    } while (0)

// Owner of `cap` elements of device (DevBuf) or pinned host (PinnedBuf) memory: move-only, freed by its destructor.
template <typename T, bool PINNED>
class Buf {
    T *p_ = nullptr;
    void release() {
        if (p_) PINNED ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        cap = 0;
    }

  public:
    int64_t cap = 0;
    Buf() = default;
    Buf(Buf &&o) noexcept : p_(o.p_), cap(o.cap) { o.p_ = nullptr; o.cap = 0; }
    Buf &operator=(Buf &&o) noexcept { std::swap(p_, o.p_); std::swap(cap, o.cap); return *this; }   // o frees the old memory
    ~Buf() { release(); }
    T *get() const { return p_; }
    operator T *() const { return p_; }
    // n elements, for a buffer of fixed size
    int alloc(int64_t n) {
        release();
        void *p = nullptr;
        const size_t bytes = (size_t)n * sizeof(T);
        CU(PINNED ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes));
        p_ = static_cast<T *>(p);
        cap = n;
        return KTA_OK;
    }
    // at least `need` elements (contents not kept): null with cap 0 if the allocation fails
    int grow(cudaStream_t s, int64_t need) {
        if (need <= cap) return KTA_OK;
        CU(cudaStreamSynchronize(s));   // queued work may still read the old buffer
        return alloc(need + need / 4 + 64);
    }
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;
