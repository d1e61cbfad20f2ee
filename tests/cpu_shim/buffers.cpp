/*
 * tests/cpu_shim/buffers.cpp — TEST-ONLY host build of the buffer and event owners (lv_buffers.h) against a fake CUDA runtime.
 *
 * The fake defines cudaMalloc, cudaMallocHost, cudaFree, cudaFreeHost, cudaEventCreateWithFlags, cudaEventDestroy and
 * cudaGetLastError.  It hands out heap memory, counts what is live, flags every free of a pointer it does not hold (a foreign
 * or a double free), and can fail the k-th allocation from now, setting the last error as the runtime does.  The library is
 * linked with -Bsymbolic, so the owners call these fakes even in a process that has loaded the real runtime.  The owners are
 * reached through opaque handles; a handle holds a device or a pinned buffer of doubles.  Not part of the product.
 */
#include <stdint.h>
#include <stdlib.h>

#include <set>
#include <utility>

#include "../../limo-velo_b200/csrc/lv_buffers.h"

using namespace lv;

namespace {
struct Fake {
    std::set<void*> device, pinned, events;
    int64_t allocs = 0, frees = 0, foreign = 0;
    int64_t fail_at = 0;                  /* the fail_at-th allocation from now fails (0: none) */
    cudaError_t last = cudaSuccess;
};
Fake g;

cudaError_t fake_alloc(std::set<void*>& live, void** p) {
    g.allocs++;
    if (g.fail_at > 0 && --g.fail_at == 0) {
        g.last = cudaErrorMemoryAllocation;
        return cudaErrorMemoryAllocation;
    }
    *p = malloc(1);
    live.insert(*p);
    return cudaSuccess;
}
cudaError_t fake_free(std::set<void*>& live, void* p) {
    if (!p) return cudaSuccess;
    if (!live.erase(p)) {
        g.foreign++;
        return cudaErrorInvalidValue;
    }
    g.frees++;
    free(p);
    return cudaSuccess;
}

struct Owner {
    bool pinned;
    DeviceBuf<double> d;
    PinnedBuf<double> h;
};
}  // namespace

extern "C" {

cudaError_t cudaMalloc(void** p, size_t) { return fake_alloc(g.device, p); }
cudaError_t cudaMallocHost(void** p, size_t) { return fake_alloc(g.pinned, p); }
cudaError_t cudaFree(void* p) { return fake_free(g.device, p); }
cudaError_t cudaFreeHost(void* p) { return fake_free(g.pinned, p); }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned int) {
    void* p = nullptr;
    const cudaError_t r = fake_alloc(g.events, &p);
    if (r == cudaSuccess) *e = static_cast<cudaEvent_t>(p);
    return r;
}
cudaError_t cudaEventDestroy(cudaEvent_t e) { return fake_free(g.events, e); }
cudaError_t cudaGetLastError(void) {
    const cudaError_t e = g.last;
    g.last = cudaSuccess;
    return e;
}

void shim_buf_fail_at(int64_t k) { g.fail_at = k; }
/* live device, pinned and event allocations, allocation calls, frees, foreign or double frees, the pending last error */
void shim_buf_counts(int64_t* out) {
    out[0] = (int64_t)g.device.size();
    out[1] = (int64_t)g.pinned.size();
    out[2] = (int64_t)g.events.size();
    out[3] = g.allocs;
    out[4] = g.frees;
    out[5] = g.foreign;
    out[6] = (int64_t)g.last;
}

void* shim_buf_new(int pinned) {
    Owner* o = new Owner();
    o->pinned = pinned != 0;
    return o;
}
void shim_buf_delete(void* o) { delete static_cast<Owner*>(o); }
int shim_buf_reserve(void* v, int64_t n) {
    Owner* o = static_cast<Owner*>(v);
    return (int)(o->pinned ? o->h.reserve((size_t)n) : o->d.reserve((size_t)n));
}
void shim_buf_reset(void* v) {
    Owner* o = static_cast<Owner*>(v);
    if (o->pinned) o->h.reset(); else o->d.reset();
}
int64_t shim_buf_size(void* v) {
    Owner* o = static_cast<Owner*>(v);
    return (int64_t)(o->pinned ? o->h.size() : o->d.size());
}
uintptr_t shim_buf_ptr(void* v) {
    Owner* o = static_cast<Owner*>(v);
    return (uintptr_t)(o->pinned ? static_cast<double*>(o->h) : static_cast<double*>(o->d));
}
/* a new handle move-constructed from src */
void* shim_buf_move_new(void* src) {
    Owner* s = static_cast<Owner*>(src);
    Owner* o = new Owner{s->pinned, std::move(s->d), std::move(s->h)};
    return o;
}
/* dst = std::move(src) (both of one kind) */
void shim_buf_move_assign(void* dst, void* src) {
    Owner* d = static_cast<Owner*>(dst);
    Owner* s = static_cast<Owner*>(src);
    if (d->pinned) d->h = std::move(s->h); else d->d = std::move(s->d);
}

void* shim_event_new() { return new Event(); }
void shim_event_delete(void* e) { delete static_cast<Event*>(e); }
int shim_event_create(void* e) { return (int)static_cast<Event*>(e)->create(); }
uintptr_t shim_event_handle(void* e) {
    const cudaEvent_t ev = *static_cast<Event*>(e);
    return (uintptr_t)ev;
}

}  // extern "C"
