// cuda_resources.h -- owners of the host runtime's CUDA resources (host code only).  Device memory, pinned host memory, events and
// streams are released by their owner's destructor, so an early return or an exception frees whatever was created before it.
#pragma once
#include "host_api.h"
#include <cuda_runtime.h>
#include <memory>
#include <type_traits>
#include <vector>

namespace b200pt {

struct DeviceFree { void operator()(void *p) const { cudaFree(p); } };
struct PinnedFree { void operator()(void *p) const { cudaFreeHost(p); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };

template <class T> using DevPtr = std::unique_ptr<T, DeviceFree>;      // cudaMalloc
template <class T> using PinnedPtr = std::unique_ptr<T, PinnedFree>;   // cudaMallocHost
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;

// p's block is released first, then p owns a new block of `bytes` (pinned host memory for a PinnedPtr, device memory otherwise), or
// nothing when the allocation fails.
template <class T, class Free> cudaError_t alloc(std::unique_ptr<T, Free> &p, size_t bytes) {
    p.reset();
    T *raw = nullptr;
    const cudaError_t e = std::is_same<Free, PinnedFree>::value ? cudaMallocHost(&raw, bytes) : cudaMalloc(&raw, bytes);
    p.reset(raw);
    return e;
}

// Device blocks that live until the list is cleared or destroyed (cudaFree waits for the work still using a block): the arrays of one
// query-hook call, the pose data of a scene, the arrays of a wave context.  in / get / sync copy and synchronise on the stream given at
// construction (the query hooks').  Each allocation, copy and synchronisation throws CudaError on failure.
class DeviceBlocks {
public:
    explicit DeviceBlocks(cudaStream_t st = nullptr) : st_(st) {}
    template <class T> T *out(size_t count) {                 // uninitialised
        T *p = nullptr;
        blocks_.emplace_back();                               // before the allocation: a full vector cannot lose the block
        check(cudaMalloc(&p, count * sizeof(T)), "cudaMalloc");
        blocks_.back().reset(p);
        return p;
    }
    template <class T> T *in(const T *src, size_t count) {    // filled from host memory
        T *p = out<T>(count);
        check(cudaMemcpyAsync(p, src, count * sizeof(T), cudaMemcpyHostToDevice, st_), "cudaMemcpyAsync");
        return p;
    }
    template <class T> void get(T *dst, const T *src, size_t count) {
        check(cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, st_), "cudaMemcpyAsync");
    }
    void sync() { check(cudaStreamSynchronize(st_), "cudaStreamSynchronize"); check(cudaGetLastError(), "cudaGetLastError"); }   // the first error
    void clear() { blocks_.clear(); }
private:
    static void check(cudaError_t e, const char *what) {
        if (e != cudaSuccess) throw CudaError{ (int)e, std::string(what) + ": " + cudaGetErrorString(e) };
    }
    cudaStream_t st_;
    std::vector<DevPtr<void>> blocks_;
};

} // namespace b200pt
