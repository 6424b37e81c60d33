// csrc/ctx_memory.h against fake CUDA allocation calls: the fakes count live allocations and record every call, and
// can fail the n-th allocation.  Run with one case name; prints "ok" when the case holds.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <map>
#include <string>
#include <vector>
#include "../../low-cost-mocap_b200/csrc/ctx_memory.h"

static std::vector<std::string> calls;          // the CUDA calls made, in order
static std::map<void*, size_t> live;            // live allocations -> bytes
static int allocs = 0, fail_alloc = -1;         // allocations made; fail the one with this index
static std::vector<unsigned char> zeroed;       // bytes cudaMemsetAsync was asked to zero, per allocation

static cudaError_t fake_alloc(void** p, size_t bytes, const char* what) {
    calls.push_back(what);
    if (allocs++ == fail_alloc) { *p = nullptr; return cudaErrorMemoryAllocation; }
    *p = malloc(bytes ? bytes : 1);
    memset(*p, 0xAB, bytes);
    live[*p] = bytes;
    return cudaSuccess;
}
static cudaError_t fake_free(void* p, const char* what) {
    calls.push_back(what);
    if (p) { if (!live.erase(p)) { printf("free of an unknown pointer\n"); exit(2); } free(p); }
    return cudaSuccess;
}

extern "C" {
cudaError_t cudaMalloc(void** p, size_t bytes) { return fake_alloc(p, bytes, "cudaMalloc"); }
cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned int flags) {
    return fake_alloc(p, bytes, flags == cudaHostAllocMapped ? "cudaHostAlloc(mapped)" : "cudaHostAlloc");
}
cudaError_t cudaFree(void* p) { return fake_free(p, "cudaFree"); }
cudaError_t cudaFreeHost(void* p) { return fake_free(p, "cudaFreeHost"); }
cudaError_t cudaMemsetAsync(void* p, int v, size_t bytes, cudaStream_t) {
    calls.push_back("cudaMemsetAsync");
    memset(p, v, bytes);
    return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { calls.push_back("cudaStreamSynchronize"); return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void) { calls.push_back("cudaDeviceSynchronize"); return cudaSuccess; }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "fake error"; }
}

struct FakeCtx {
    cudaStream_t stream = nullptr;
    char err[256] = {0};
    DeviceBuffer a, b;
    PinnedBuffer h, m;
};
int mocap_fail(FakeCtx* ctx, int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
    va_end(ap);
    return code;
}

#define CHECK(c) do { if (!(c)) { printf("FAILED line %d: %s\n", __LINE__, #c); return 1; } } while (0)
static std::vector<std::string> seq(std::initializer_list<const char*> l) { return std::vector<std::string>(l.begin(), l.end()); }

static int no_call_when_big_enough() {
    FakeCtx ctx;
    CHECK(ctx.a.grow(&ctx, 1000, Drain::stream) == MOCAP_OK && ctx.a.bytes() == 1000);
    void* p = ctx.a.get();
    calls.clear();
    CHECK(ctx.a.grow(&ctx, 1000, Drain::stream) == MOCAP_OK);
    CHECK(ctx.a.grow(&ctx, 10, Drain::device, 10) == MOCAP_OK);
    CHECK(ctx.h.grow(&ctx, 0, Drain::stream) == MOCAP_OK);
    CHECK(calls.empty() && ctx.a.get() == p && ctx.a.bytes() == 1000);
    return 0;
}

static int drains_before_it_frees() {
    FakeCtx ctx;
    CHECK(ctx.a.grow(&ctx, 100, Drain::none) == MOCAP_OK);
    CHECK(calls == seq({"cudaMalloc"}));
    calls.clear();
    CHECK(ctx.a.grow(&ctx, 200, Drain::stream) == MOCAP_OK);
    CHECK(calls == seq({"cudaStreamSynchronize", "cudaFree", "cudaMalloc"}));
    calls.clear();
    CHECK(ctx.a.grow(&ctx, 300, Drain::device) == MOCAP_OK);
    CHECK(calls == seq({"cudaDeviceSynchronize", "cudaFree", "cudaMalloc"}));
    calls.clear();
    CHECK(ctx.h.grow(&ctx, 64, Drain::stream, 0, cudaHostAllocMapped) == MOCAP_OK);
    CHECK(ctx.h.grow(&ctx, 128, Drain::device) == MOCAP_OK);
    CHECK(calls == seq({"cudaStreamSynchronize", "cudaHostAlloc(mapped)", "cudaDeviceSynchronize", "cudaFreeHost", "cudaHostAlloc"}));
    CHECK(ctx.a.bytes() == 300 && ctx.h.bytes() == 128 && live.size() == 2);
    return 0;
}

static int zero_fill_covers_the_new_allocation() {
    FakeCtx ctx;
    CHECK(ctx.a.grow(&ctx, 4096, Drain::stream, 4096) == MOCAP_OK);
    for (size_t i = 0; i < 4096; ++i) CHECK(ctx.a.as<unsigned char>()[i] == 0);
    CHECK(ctx.b.grow(&ctx, 4096, Drain::stream, 512) == MOCAP_OK);      // a zeroed prefix only
    for (size_t i = 0; i < 4096; ++i) CHECK(ctx.b.as<unsigned char>()[i] == (i < 512 ? 0 : 0xAB));
    CHECK(ctx.m.grow(&ctx, 16, Drain::none, 16, cudaHostAllocMapped) == MOCAP_OK);    // pinned: zeroed on the host
    for (size_t i = 0; i < 16; ++i) CHECK(ctx.m.as<unsigned char>()[i] == 0);
    CHECK(ctx.a.grow(&ctx, 8192, Drain::stream, 8192) == MOCAP_OK);
    for (size_t i = 0; i < 8192; ++i) CHECK(ctx.a.as<unsigned char>()[i] == 0);
    return 0;
}

static int failed_allocation_leaves_it_empty() {
    FakeCtx ctx;
    CHECK(ctx.a.grow(&ctx, 100, Drain::none) == MOCAP_OK);
    fail_alloc = allocs;
    CHECK(ctx.a.grow(&ctx, 200, Drain::stream) == MOCAP_ECUDA);
    CHECK(ctx.a.get() == nullptr && ctx.a.bytes() == 0 && live.empty() && strstr(ctx.err, "200 bytes"));
    CHECK(ctx.a.grow(&ctx, 200, Drain::stream) == MOCAP_OK);               // the retry allocates
    CHECK(ctx.a.get() != nullptr && ctx.a.bytes() == 200 && live.size() == 1);
    fail_alloc = allocs;
    CHECK(ctx.h.grow(&ctx, 64, Drain::none) == MOCAP_ECUDA && ctx.h.get() == nullptr && ctx.h.bytes() == 0);
    CHECK(ctx.h.grow(&ctx, 64, Drain::none) == MOCAP_OK && ctx.h.bytes() == 64);
    return 0;
}

static int destroying_the_owner_frees_everything() {
    {
        FakeCtx ctx;
        CHECK(ctx.a.grow(&ctx, 100, Drain::none) == MOCAP_OK && ctx.b.grow(&ctx, 5000, Drain::none, 5000) == MOCAP_OK);
        CHECK(ctx.h.grow(&ctx, 300, Drain::none) == MOCAP_OK && ctx.m.grow(&ctx, 16, Drain::none, 16, cudaHostAllocMapped) == MOCAP_OK);
        CHECK(ctx.a.grow(&ctx, 900, Drain::stream) == MOCAP_OK && live.size() == 4);
    }
    CHECK(live.empty());
    return 0;
}

// a layout of mixed types and sizes (zero-sized regions included), zeroed up to the third region
struct Regions { double* d; uint8_t* u; int32_t* i; uint8_t* empty; unsigned long long* w; };
static void declare(Layout& L, Regions& r, size_t n) {
    r.d = L.take<double>(3 * n); r.u = L.take<uint8_t>(n + 1); r.i = L.take<int32_t>(n);
    L.zero_so_far();
    r.empty = L.take<uint8_t>(0); r.w = L.take<unsigned long long>(2 * n + 7);
}

static int layout_is_aligned_ordered_and_sized_once() {
    for (size_t n : {1, 5, 64, 1000, 12345}) {
        Layout size;
        Regions r;
        declare(size, r, n);
        CHECK(r.d == nullptr && r.w == nullptr);                       // sizing hands out no pointers
        CHECK(size.bytes() % 256 == 0 && size.zeroed() % 256 == 0 && size.zeroed() <= size.bytes());
        std::vector<unsigned char> mem(size.bytes() + 256);
        unsigned char* base = mem.data() + (256 - reinterpret_cast<uintptr_t>(mem.data()) % 256) % 256;
        Layout carve(base);
        declare(carve, r, n);
        CHECK(carve.bytes() == size.bytes() && carve.zeroed() == size.zeroed());
        const size_t off[] = {(size_t)((uint8_t*)r.d - base), (size_t)(r.u - base), (size_t)((uint8_t*)r.i - base),
                              (size_t)(r.empty - base), (size_t)((uint8_t*)r.w - base)};
        const size_t len[] = {3 * n * 8, n + 1, n * 4, 0, (2 * n + 7) * 8};
        CHECK(off[0] == 0);
        for (int k = 0; k < 5; ++k) {
            CHECK(off[k] % 256 == 0);
            if (k) CHECK(off[k] >= off[k - 1] + len[k - 1]);            // in order, disjoint
        }
        CHECK(off[4] + len[4] <= size.bytes() && size.bytes() - (off[4] + len[4]) < 256);
        CHECK(size.zeroed() == off[3] && size.zeroed() >= off[2] + len[2]);
    }
    FakeCtx ctx;                                                        // grow_carved: one allocation, zeroed prefix
    Regions r;
    CHECK(grow_carved(&ctx, ctx.a, Drain::stream, [&](Layout& L) { declare(L, r, 100); }) == MOCAP_OK);
    CHECK(ctx.a.get() == (void*)r.d && calls == seq({"cudaStreamSynchronize", "cudaMalloc", "cudaMemsetAsync"}));
    for (size_t i = 0; i < (size_t)((uint8_t*)r.i - (uint8_t*)r.d) + 400; ++i) CHECK(ctx.a.as<unsigned char>()[i] == 0);
    calls.clear();
    CHECK(grow_carved(&ctx, ctx.a, Drain::stream, [&](Layout& L) { declare(L, r, 50); }) == MOCAP_OK);
    CHECK(calls.empty() && ctx.a.get() == (void*)r.d);
    return 0;
}

int main(int argc, char** argv) {
    const std::map<std::string, int (*)()> cases = {
        {"no_call_when_big_enough", no_call_when_big_enough},
        {"drains_before_it_frees", drains_before_it_frees},
        {"zero_fill_covers_the_new_allocation", zero_fill_covers_the_new_allocation},
        {"failed_allocation_leaves_it_empty", failed_allocation_leaves_it_empty},
        {"destroying_the_owner_frees_everything", destroying_the_owner_frees_everything},
        {"layout_is_aligned_ordered_and_sized_once", layout_is_aligned_ordered_and_sized_once},
    };
    if (argc != 2 || !cases.count(argv[1])) { printf("unknown case\n"); return 2; }
    const int r = cases.at(argv[1])();
    if (r == 0) printf("ok\n");
    return r;
}
