// The device and page-locked memory a mocap_ctx owns.  Host code only: kernels never see these types.
//
// Every allocation is a CtxBuffer: it frees itself, and it changes size one way only, grow() (at least this many bytes,
// or nothing at all).  An allocation that holds several arrays is described once by a Layout, which sizes it and then
// carves it.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "../../include/mocap_b200.h"

// What grow() waits for before it frees a buffer that is too small: the work queued on the context's stream, the
// whole device (buffers the copy streams use as well), or nothing (the caller has synchronised, or nothing can use it).
enum class Drain { none, stream, device };

inline size_t round_up(size_t bytes, size_t to) { return (bytes + to - 1) / to * to; }

template <bool Pinned>
class CtxBuffer {
public:
    CtxBuffer() = default;
    CtxBuffer(const CtxBuffer&) = delete;
    CtxBuffer& operator=(const CtxBuffer&) = delete;
    ~CtxBuffer() { reset(); }

    void* get() const { return p_; }
    template <class T> T* as() const { return static_cast<T*>(p_); }
    size_t bytes() const { return bytes_; }

    // frees the allocation; the caller makes sure nothing queued still uses it
    void reset() {
        if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        bytes_ = 0;
    }

    // At least `bytes`.  A buffer that holds that much already is left as it is, without a CUDA call.  Otherwise:
    // drain, free, allocate, and zero the first `zero` bytes of the new allocation (device: on ctx->stream).  If the
    // drain fails the buffer is kept; if the allocation or the zeroing fails the buffer is left empty, so the next call
    // tries again.  Failures return MOCAP_ECUDA through mocap_fail.  flags: cudaHostAlloc's (pinned only).
    template <class Ctx>
    int grow(Ctx* ctx, size_t bytes, Drain drain, size_t zero = 0, unsigned flags = cudaHostAllocDefault) {
        if (bytes <= bytes_) return MOCAP_OK;
        cudaError_t e = drain == Drain::stream ? cudaStreamSynchronize(ctx->stream)
                      : drain == Drain::device ? cudaDeviceSynchronize() : cudaSuccess;
        if (e != cudaSuccess) return mocap_fail(ctx, MOCAP_ECUDA, "synchronisation before a buffer grows: %s", cudaGetErrorString(e));
        reset();
        void* p = nullptr;
        e = Pinned ? cudaHostAlloc(&p, bytes, flags) : cudaMalloc(&p, bytes);
        if (e == cudaSuccess) p_ = p;
        if (e == cudaSuccess && zero) {
            if (Pinned) memset(p_, 0, zero);
            else e = cudaMemsetAsync(p_, 0, zero, ctx->stream);
        }
        if (e != cudaSuccess) {
            cudaGetLastError();
            reset();
            return mocap_fail(ctx, MOCAP_ECUDA, "%zu bytes of %s memory: %s", bytes, Pinned ? "page-locked" : "device", cudaGetErrorString(e));
        }
        bytes_ = bytes;
        return MOCAP_OK;
    }

private:
    void* p_ = nullptr;
    size_t bytes_ = 0;
};

using DeviceBuffer = CtxBuffer<false>;
using PinnedBuffer = CtxBuffer<true>;

// The regions of one allocation, declared once and run twice: over no base to size the allocation, then over its
// base to carve the pointers.  Regions are 256-byte aligned and placed in declaration order, the first at offset 0.
class Layout {
public:
    explicit Layout(void* base = nullptr) : base_(static_cast<uint8_t*>(base)) {}

    // a region of `count` T (nullptr while sizing)
    template <class T> T* take(size_t count) {
        const size_t at = end_;
        end_ += round_up(count * sizeof(T), 256);
        return base_ ? reinterpret_cast<T*>(base_ + at) : nullptr;
    }
    // the regions declared so far are zeroed when the allocation is new (so zeroed regions come first)
    void zero_so_far() { zero_ = end_; }

    size_t bytes() const { return end_; }
    size_t zeroed() const { return zero_; }

private:
    uint8_t* base_;
    size_t end_ = 0, zero_ = 0;
};

// Sizes the layout `regions(Layout&)` declares, grows `buf` to hold it and carves `buf` by it.  `regions` runs twice
// and must declare the same regions both times.
template <class Ctx, class Regions>
int grow_carved(Ctx* ctx, DeviceBuffer& buf, Drain drain, Regions&& regions) {
    Layout size;
    regions(size);
    const int st = buf.grow(ctx, size.bytes(), drain, size.zeroed());
    if (st) return st;
    Layout carve(buf.get());
    regions(carve);
    return MOCAP_OK;
}
