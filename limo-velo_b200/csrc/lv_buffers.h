/*
 * lv_buffers.h — owners of device buffers, pinned host buffers and events (host code only).
 *
 * A context keeps many buffers that are allocated at create time or on first use and that some calls grow.  Each owner frees
 * its allocation exactly once, in its destructor or when it grows, so no code keeps a list of what to free.  An allocation
 * that fails leaves its owner empty: the next call that needs the buffer allocates it again instead of using a freed or
 * missing pointer.  The failure is also cleared from the runtime's last error, so that a later launcher that returns
 * cudaGetLastError() does not report it as its own.
 */
#ifndef LV_BUFFERS_H_
#define LV_BUFFERS_H_

#include <cuda_runtime_api.h>
#include <stddef.h>

namespace lv {

/* n elements of T in device memory or in pinned host memory; move-only (declaring the move deletes the copies), and converts
 * to T* so that it reads as the pointer it owns */
template <class T, bool Pinned>
class Buffer {
public:
    Buffer() = default;
    Buffer(Buffer&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    Buffer& operator=(Buffer&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_; n_ = o.n_;
            o.p_ = nullptr; o.n_ = 0;
        }
        return *this;
    }
    ~Buffer() { reset(); }

    /* grow-only: nothing happens when n elements fit; otherwise the old allocation is freed first, then exactly n elements
     * are allocated.  On failure the buffer is left empty and the runtime's last error is cleared. */
    cudaError_t reserve(size_t n) {
        if (n <= n_) return cudaSuccess;
        reset();
        void* q = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&q, sizeof(T) * n) : cudaMalloc(&q, sizeof(T) * n);
        if (e != cudaSuccess) { cudaGetLastError(); return e; }
        p_ = static_cast<T*>(q);
        n_ = n;
        return cudaSuccess;
    }
    void reset() {
        if (p_) (void)(Pinned ? cudaFreeHost(p_) : cudaFree(p_));
        p_ = nullptr;
        n_ = 0;
    }
    size_t size() const { return n_; }
    T* get() const { return p_; }      /* for template arguments, where the conversion is not deduced */
    operator T*() const { return p_; }
    T* operator->() const { return p_; }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <class T> using DeviceBuf = Buffer<T, false>;
template <class T> using PinnedBuf = Buffer<T, true>;

/* a cudaEventDisableTiming event, created by the first create() that succeeds and destroyed with its owner */
class Event {
public:
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (e_) cudaEventDestroy(e_); }
    cudaError_t create() {
        if (e_) return cudaSuccess;
        const cudaError_t e = cudaEventCreateWithFlags(&e_, cudaEventDisableTiming);
        if (e != cudaSuccess) { e_ = nullptr; cudaGetLastError(); }
        return e;
    }
    operator cudaEvent_t() const { return e_; }

private:
    cudaEvent_t e_ = nullptr;
};

}  // namespace lv
#endif
