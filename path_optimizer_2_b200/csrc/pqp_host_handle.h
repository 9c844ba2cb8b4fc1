// pqp_host_handle.h — host plumbing shared by the library's C-ABI handles: the device guard, the error path of
// an entry point, and the owner of a handle's CUDA resources. No device code here.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <string>
#include <vector>

#include "../../include/pqp.h"

namespace pqp {

// every handle of the library is bound to one CUDA device; an API call switches to it for its own duration and
// leaves the caller's current device as it found it
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
};

// `slot` is a handle's `err`, or its ABI's create-error string when there is no handle yet
inline int fail(std::string &slot, int code, const std::string &msg) {
    slot = msg;
    return code;
}

// a failed CUDA runtime call returns PQP_E_CUDA from the enclosing function, "<call>: <error string>" in `slot`
#define PQP_CUDA(slot, call)                                                                                      \
    do {                                                                                                          \
        const cudaError_t e_ = (call);                                                                            \
        if (e_ != cudaSuccess) return ::pqp::fail((slot), PQP_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

// The CUDA resources of one handle on one device. Each device buffer (one cudaMalloc per buffer), pinned or mapped
// host buffer, stream and event is made through the owner into the handle member that holds it; the owner records
// that member, so a handle lists each resource in its struct and at its one allocation site only. The destructor
// frees everything exactly once, newest first, under the device's guard, and clears the members; a failed
// all-or-nothing group frees its own part the same way.
class Resources {
public:
    int device = 0;

    Resources() = default;
    Resources(const Resources &) = delete;
    Resources &operator=(const Resources &) = delete;
    ~Resources() { release(0); }

    template <typename T>
    cudaError_t alloc(T *&p, size_t count) {
        return alloc(reinterpret_cast<void *&>(p), count * sizeof(T));
    }
    // an untyped device buffer (a handle option picks its element type): `bytes`, not a count
    cudaError_t alloc(void *&p, size_t bytes) { return add(kDevice, &p, bytes, cudaMalloc(&p, bytes)); }
    // pinned host memory; cudaHostAllocMapped for memory the device writes through its alias
    template <typename T>
    cudaError_t alloc_host(T *&p, size_t count, unsigned flags = cudaHostAllocDefault) {
        return add(kHost, reinterpret_cast<void **>(&p), 0, cudaHostAlloc(reinterpret_cast<void **>(&p), count * sizeof(T), flags));
    }
    cudaError_t stream(cudaStream_t &s) {
        return add(kStream, reinterpret_cast<void **>(&s), 0, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    }
    cudaError_t event(cudaEvent_t &e, unsigned flags = cudaEventDefault) {
        return add(kEvent, reinterpret_cast<void **>(&e), 0, cudaEventCreateWithFlags(&e, flags));
    }
    // a device buffer grown on demand: a request for more than `p` holds replaces it with a buffer of `count`; after a
    // failure `p` is null, so the next request allocates again
    template <typename T>
    cudaError_t grow(T *&p, size_t count) {
        for (size_t i = 0; i < items_.size(); ++i)
            if (items_[i].slot == reinterpret_cast<void **>(&p)) {
                if (count * sizeof(T) <= items_[i].bytes) return cudaSuccess;
                destroy(items_[i]);
                items_.erase(items_.begin() + (std::ptrdiff_t)i);
                break;
            }
        return alloc(p, count);
    }
    // all or nothing: if `allocate` (a sequence of this owner's calls) fails, whatever it made is released
    template <typename F>
    cudaError_t group(F &&allocate) {
        const size_t mark = items_.size();
        const cudaError_t e = allocate();
        if (e != cudaSuccess) release(mark);
        return e;
    }

private:
    enum Kind { kDevice, kHost, kStream, kEvent };
    struct Item {
        Kind kind;
        void **slot;
        size_t bytes;  // of a device buffer
    };
    std::vector<Item> items_;

    cudaError_t add(Kind kind, void **slot, size_t bytes, cudaError_t e) {
        if (e == cudaSuccess) items_.push_back({kind, slot, bytes});
        else *slot = nullptr;
        return e;
    }
    static void destroy(const Item &it) {
        switch (it.kind) {
            case kDevice: cudaFree(*it.slot); break;
            case kHost: cudaFreeHost(*it.slot); break;
            case kStream: cudaStreamDestroy(static_cast<cudaStream_t>(*it.slot)); break;
            case kEvent: cudaEventDestroy(static_cast<cudaEvent_t>(*it.slot)); break;
        }
        *it.slot = nullptr;
    }
    void release(size_t mark) {
        if (items_.size() <= mark) return;
        DeviceGuard guard_(device);
        while (items_.size() > mark) {
            destroy(items_.back());
            items_.pop_back();
        }
    }
};

}  // namespace pqp
