// Owners for the CUDA resources the shim holds (fabgpu_shim.cu): each frees its resource when it goes out of scope or is replaced.
// Nothing else of the runtime is wrapped here: copies, launches and stream-ordered allocations are called directly.
#pragma once
#include <cuda_runtime.h>

#include <cstdio>
#include <memory>
#include <type_traits>
#include <utility>

#include "../../include/fabgpu_ecdsa.h"

namespace fabgpu {

// An array of T in device memory (Pinned = false) or in pinned, portable host memory (Pinned = true).  Move-only.
template <typename T, bool Pinned>
class CudaArray {
public:
    CudaArray() = default;
    CudaArray(CudaArray&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
    CudaArray& operator=(CudaArray&& o) noexcept
    {
        if (this != &o) { release(); p_ = std::exchange(o.p_, nullptr); bytes_ = std::exchange(o.bytes_, 0); }
        return *this;
    }
    ~CudaArray() { release(); }

    T* get() const { return p_; }
    size_t bytes() const { return bytes_; }     // size of the allocation, 0 when there is none

    // Makes the array at least `bytes` long.  A shorter array is freed before the new one is allocated, so growing never holds both
    // (contents are not kept).  On failure the array is empty and ctx->last_error says why.
    template <typename Ctx>
    int reserve(Ctx* ctx, size_t bytes)
    {
        if (bytes <= bytes_) return FABGPU_OK;
        release();
        void* p = nullptr;
        const cudaError_t e = Pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocPortable) : cudaMalloc(&p, bytes);
        if (e != cudaSuccess) {
            char buf[256];
            snprintf(buf, sizeof buf, "%s(%zu bytes) failed: %s", Pinned ? "cudaHostAlloc" : "cudaMalloc", bytes, cudaGetErrorString(e));
            ctx->last_error = buf;
            return FABGPU_E_CUDA;
        }
        p_ = static_cast<T*>(p);
        bytes_ = bytes;
        return FABGPU_OK;
    }

private:
    void release()
    {
        if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr;
        bytes_ = 0;
    }
    T* p_ = nullptr;
    size_t bytes_ = 0;
};
template <typename T> using DevArray = CudaArray<T, false>;
template <typename T> using HostArray = CudaArray<T, true>;

struct StreamDeleter { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct EventDeleter { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct MemPoolDeleter { void operator()(cudaMemPool_t p) const { cudaMemPoolDestroy(p); } };   // frees still in flight complete on their own
struct IpcDeleter { void operator()(void* p) const { cudaIpcCloseMemHandle(p); } };
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDeleter>;
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDeleter>;
using MemPool = std::unique_ptr<std::remove_pointer_t<cudaMemPool_t>, MemPoolDeleter>;
template <typename T> using IpcMapping = std::unique_ptr<T, IpcDeleter>;    // a peer's buffer opened with cudaIpcOpenMemHandle

}  // namespace fabgpu
