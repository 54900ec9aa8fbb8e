// TEST INFRASTRUCTURE: what the GPU probes under tests/native/ share — a CUDA call that fails ends the program (exit 3),
// stdin / stdout in raw bytes (a short read exits 2, a short write 4), and device buffers that are allocated filled with one
// byte (so an entry a pass does not write shows up) and read back.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(call)                                                                                           \
    do {                                                                                                   \
        cudaError_t e_ = (call);                                                                           \
        if (e_ != cudaSuccess) {                                                                           \
            fprintf(stderr, "%s: %s (%s:%d)\n", #call, cudaGetErrorString(e_), __FILE__, __LINE__);        \
            exit(3);                                                                                       \
        }                                                                                                  \
    } while (0)

inline void put(const void *p, size_t n) {
    if (n && fwrite(p, 1, n, stdout) != n) exit(4);
}

inline void get(void *p, size_t n) {
    if (n && fread(p, 1, n, stdin) != n) exit(2);
}

// count elements (at least one), every byte `fill`
template <typename T>
inline T *dev_alloc(size_t count, int fill, cudaStream_t s) {
    T *p = nullptr;
    CK(cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T)));
    CK(cudaMemsetAsync(p, fill, std::max<size_t>(count, 1) * sizeof(T), s));
    return p;
}

template <typename T>
inline std::vector<T> from_dev(const T *d, size_t count) {
    std::vector<T> h(count);
    if (count) CK(cudaMemcpy(h.data(), d, count * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}

template <typename T>
inline void put_dev(const T *d, size_t count) {
    put(from_dev(d, count).data(), count * sizeof(T));
}
