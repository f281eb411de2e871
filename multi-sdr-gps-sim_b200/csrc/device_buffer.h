// Device buffers grown to what a call needs, and the error return of host code that reports cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

// Return the error of a CUDA call from a function that returns cudaError_t.
#define CU_RET(call)                      \
    do {                                  \
        cudaError_t e_ = (call);          \
        if (e_ != cudaSuccess) return e_; \
    } while (0)

namespace gpsb200 {

// Make p hold at least n elements of T; cap is its size in elements. A larger buffer replaces the old one without its
// contents. On a failed allocation p is NULL and cap 0.
template <typename T>
cudaError_t grow(T *&p, size_t &cap, size_t n) {
    if (n <= cap) return cudaSuccess;
    cudaFree(p);
    p = nullptr;
    cap = 0;
    CU_RET(cudaMalloc(&p, n * sizeof(T)));
    cap = n;
    return cudaSuccess;
}

}  // namespace gpsb200
