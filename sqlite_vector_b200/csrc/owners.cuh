// owners.cuh — move-only owners of the CUDA resources the host engine holds: device and pinned allocations, events, streams
// and IPC mappings.  An owner releases its handle when it is destroyed, reset, or given a new one; the rest of the host code
// never calls a release function itself.
//
// Lifetime rules:
//  - An object that holds owners is destroyed only after its streams are drained and with its device current: a release acts on
//    the current device, and an event or stream may not be destroyed under work that still uses it.
//  - Streams are declared first in such an object, so they are destroyed last.
//  - No owner lives in a static or global object: with -cudart static the runtime may be torn down before static destructors run.
//  - A buffer that an in-flight batch may still read is regrown only behind the synchronisation that guards it.
//  - A group of resources built on first need is allocated into local owners and moved into its object only when every
//    allocation has succeeded: after a failure the object is as it was, and the next call retries.
#pragma once

#include <cuda_runtime.h>

#include <atomic>

namespace vsb {

// owned handles alive in this process (vsb_debug_live_handles); atomic because several host threads allocate at once (the
// streamed shards of a group each run on their own thread)
inline std::atomic<long long> g_live_handles{0};

// Rel::release(H) gives the handle back to the runtime
template <class H, class Rel>
class Owner {
public:
    Owner() = default;
    Owner(const Owner &) = delete;
    Owner &operator=(const Owner &) = delete;
    Owner(Owner &&o) noexcept : h_(o.h_) { o.h_ = H(); }
    Owner &operator=(Owner &&o) noexcept {
        if (this != &o) {
            reset();
            h_ = o.h_;
            o.h_ = H();
        }
        return *this;
    }
    ~Owner() { reset(); }

    H get() const { return h_; }
    operator H() const { return h_; }   // an owner passes as the raw handle wherever the runtime or a kernel takes one
    void reset() {
        if (!h_) return;
        Rel::release(h_);
        h_ = H();
        --g_live_handles;
    }

protected:
    // releases the current handle first; takes the one make(&h) creates only when make succeeds, so that the owner is empty
    // after a failure
    template <class Make>
    cudaError_t acquire(Make make) {
        reset();
        H h = H();
        const cudaError_t e = make(&h);
        if (e == cudaSuccess && h) {
            h_ = h;
            ++g_live_handles;
        }
        return e;
    }

private:
    H h_ = H();
};

struct DeviceRelease { static void release(void *p) { cudaFree(p); } };
struct HostRelease { static void release(void *p) { cudaFreeHost(p); } };
struct EventRelease { static void release(cudaEvent_t e) { cudaEventDestroy(e); } };
struct StreamRelease { static void release(cudaStream_t s) { cudaStreamDestroy(s); } };
struct IpcRelease { static void release(void *p) { cudaIpcCloseMemHandle(p); } };

template <class T>
struct DeviceBuf : Owner<T *, DeviceRelease> {
    cudaError_t alloc(size_t bytes) { return this->acquire([&](T **p) { return cudaMalloc((void **)p, bytes); }); }
};

template <class T>
struct HostBuf : Owner<T *, HostRelease> {   // pinned
    cudaError_t alloc(size_t bytes) { return this->acquire([&](T **p) { return cudaHostAlloc((void **)p, bytes, cudaHostAllocDefault); }); }
};

struct Event : Owner<cudaEvent_t, EventRelease> {
    cudaError_t create(unsigned flags) { return acquire([&](cudaEvent_t *e) { return cudaEventCreateWithFlags(e, flags); }); }
};

struct Stream : Owner<cudaStream_t, StreamRelease> {   // every stream of the engine is non-blocking
    cudaError_t create() { return acquire([](cudaStream_t *s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }); }
};

struct IpcMapping : Owner<void *, IpcRelease> {   // a peer process's allocation mapped into this one
    cudaError_t open(cudaIpcMemHandle_t h, unsigned flags) { return acquire([&](void **p) { return cudaIpcOpenMemHandle(p, h, flags); }); }
};

}  // namespace vsb
