// Owning arrays of device and page-locked host memory, grown to what a call needs, and the error return of host code
// that reports cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <utility>

// Return the error of a CUDA call from a function that returns cudaError_t.
#define CU_RET(call)                      \
    do {                                  \
        cudaError_t e_ = (call);          \
        if (e_ != cudaSuccess) return e_; \
    } while (0)

namespace gpsb200 {

// n elements of T in cudaMalloc memory, freed with the array (on the device that is current then).
template <typename T>
class DeviceArray {
public:
    DeviceArray() = default;
    DeviceArray(DeviceArray &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    DeviceArray &operator=(DeviceArray &&o) noexcept {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~DeviceArray() {
        if (p_) cudaFree(p_);
    }

    // Hold at least n elements. A larger buffer replaces the old one without its contents. On a failed allocation
    // get() is NULL and size() 0.
    cudaError_t grow(size_t n) {
        if (n <= n_) return cudaSuccess;
        *this = DeviceArray();
        T *p = nullptr;
        CU_RET(cudaMalloc(&p, n * sizeof(T)));
        p_ = p;
        n_ = n;
        return cudaSuccess;
    }
    T *get() const { return p_; }
    size_t size() const { return n_; }

private:
    T *p_ = nullptr;
    size_t n_ = 0;
};

// n elements of T in cudaHostAlloc memory, freed with the array. With cudaHostAllocMapped, dev() is the device's
// address of the same memory (NULL otherwise).
template <typename T>
class PinnedArray {
public:
    PinnedArray() = default;
    PinnedArray(PinnedArray &&o) noexcept
        : p_(std::exchange(o.p_, nullptr)), d_(std::exchange(o.d_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    PinnedArray &operator=(PinnedArray &&o) noexcept {
        std::swap(p_, o.p_);
        std::swap(d_, o.d_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~PinnedArray() {
        if (p_) cudaFreeHost(p_);
    }

    // As DeviceArray::grow, allocated with cudaHostAlloc's flags.
    cudaError_t grow(size_t n, unsigned flags = cudaHostAllocDefault) {
        if (n <= n_) return cudaSuccess;
        *this = PinnedArray();
        T *p = nullptr, *d = nullptr;
        CU_RET(cudaHostAlloc((void **) &p, n * sizeof(T), flags));
        if (flags & cudaHostAllocMapped) {
            const cudaError_t e = cudaHostGetDevicePointer((void **) &d, p, 0);
            if (e != cudaSuccess) {
                cudaFreeHost(p);
                return e;
            }
        }
        p_ = p;
        d_ = d;
        n_ = n;
        return cudaSuccess;
    }
    T *get() const { return p_; }
    T &operator[](size_t i) const { return p_[i]; }
    T *dev() const { return d_; }
    size_t size() const { return n_; }

private:
    T *p_ = nullptr, *d_ = nullptr;
    size_t n_ = 0;
};

}  // namespace gpsb200
