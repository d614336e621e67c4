// Move-only owners of the engine's CUDA allocations, events, streams and graphs. Each starts null, releases what it holds in its
// destructor and in reset(), and reads as the raw pointer or handle. Allocation returns the cudaError_t and leaves the owner null on
// failure, so a set built into locals and moved into place only when every call succeeded is never half built.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <utility>

namespace rwkv {

template <class H, auto Release> class CudaOwner {
public:
    CudaOwner() = default;
    CudaOwner(CudaOwner && o) noexcept : h_(std::exchange(o.h_, H{})) {}
    CudaOwner & operator=(CudaOwner && o) noexcept {
        if (this != &o) { reset(); h_ = std::exchange(o.h_, H{}); }
        return *this;
    }
    CudaOwner(const CudaOwner &) = delete;
    CudaOwner & operator=(const CudaOwner &) = delete;
    ~CudaOwner() { reset(); }
    void reset() { if (h_) Release(std::exchange(h_, H{})); }
    H get() const { return h_; }
    operator H() const { return h_; }

protected:
    template <class Make> cudaError_t acquire(Make make) {
        reset();
        H h{};
        const cudaError_t e = make(&h);
        if (e == cudaSuccess) h_ = h;
        return e;
    }
    H h_{};
};

// cudaMalloc of `bytes` bytes.
template <class T> struct DeviceBuffer : CudaOwner<T *, cudaFree> {
    cudaError_t alloc(size_t bytes) { return this->acquire([&](T ** p) { return cudaMalloc(reinterpret_cast<void **>(p), bytes); }); }
};

// Pinned host memory of `bytes` bytes. A mapped buffer also keeps the device address it is seen at (device()).
template <class T> class PinnedBuffer : public CudaOwner<T *, cudaFreeHost> {
public:
    cudaError_t alloc(size_t bytes) { return this->acquire([&](T ** p) { return cudaMallocHost(reinterpret_cast<void **>(p), bytes); }); }
    cudaError_t alloc_mapped(size_t bytes) {
        cudaError_t e = this->acquire([&](T ** p) { return cudaHostAlloc(reinterpret_cast<void **>(p), bytes, cudaHostAllocMapped); });
        if (e == cudaSuccess) e = cudaHostGetDevicePointer(reinterpret_cast<void **>(&dev_), this->h_, 0);
        if (e != cudaSuccess) this->reset();
        return e;
    }
    T * device() const { return this->h_ ? dev_ : nullptr; }

private:
    T * dev_ = nullptr;
};

struct Event : CudaOwner<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags = cudaEventDefault) { return acquire([&](cudaEvent_t * e) { return cudaEventCreateWithFlags(e, flags); }); }
};

struct Stream : CudaOwner<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { return acquire([](cudaStream_t * s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }); }
};

struct Graph : CudaOwner<cudaGraph_t, cudaGraphDestroy> {
    cudaError_t create() { return acquire([](cudaGraph_t * g) { return cudaGraphCreate(g, 0); }); }
    cudaError_t end_capture(cudaStream_t s) { return acquire([&](cudaGraph_t * g) { return cudaStreamEndCapture(s, g); }); }
};

struct GraphExec : CudaOwner<cudaGraphExec_t, cudaGraphExecDestroy> {
    cudaError_t instantiate(cudaGraph_t g) { return acquire([&](cudaGraphExec_t * x) { return cudaGraphInstantiate(x, g, 0); }); }
};

}  // namespace rwkv
