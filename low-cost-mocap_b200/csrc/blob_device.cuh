// Device-side pieces of S1 shared by the split kernels (blob_kernels.cu) and the fused pipeline
// kernel (fused_kernel.cu): SWAR threshold, segment append, and the sparse per-image reduction
// (sort, runs, union-find, 2x2-cell polygon moments).  See blob_kernels.cu for the semantics.
#pragma once
#include "common.cuh"
#include "blob_holes.cuh"

#define SEG_PAD 0xFFFFFFFFu

// ---------------------------------------------------------------------------------------------
// threshold helpers
// ---------------------------------------------------------------------------------------------
struct ThreshConst { uint32_t addc; uint32_t use_and; };   // see swar_gt()

// bit 7 of every byte of the result is (byte > threshold).  T1 = threshold+1 in 1..255:
//   T1 <= 128:  b >= T1  <=>  high bit set  OR  low7 + (128-T1) carries into bit 7
//   T1 >  128:  b >= T1  <=>  high bit set  AND low7 + (256-T1) carries into bit 7
__device__ __forceinline__ uint32_t swar_gt(uint32_t w, ThreshConst tc) {
    uint32_t s = (w & 0x7f7f7f7fu) + tc.addc;
    return tc.use_and ? (s & w) : (s | w);
}
// "does any of the 16 bytes exceed the threshold?" -- the test every streamed 128-bit word goes through.
// OR regime (threshold < 128): bit 7 of (s | w) over the four words = bit 7 of (OR of the s) | (OR of the w),
// so the four ORs are shared: 13 integer ops per 16 pixels.
template <bool USE_AND>
__device__ __forceinline__ bool any_above(const uint4& x, ThreshConst tc) {
    const uint32_t s0 = (x.x & 0x7f7f7f7fu) + tc.addc, s1 = (x.y & 0x7f7f7f7fu) + tc.addc;
    const uint32_t s2 = (x.z & 0x7f7f7f7fu) + tc.addc, s3 = (x.w & 0x7f7f7f7fu) + tc.addc;
    if (USE_AND) return (((s0 & x.x) | (s1 & x.y) | (s2 & x.z) | (s3 & x.w)) & 0x80808080u) != 0;
    return (((s0 | s1 | s2 | s3) | (x.x | x.y | x.z | x.w)) & 0x80808080u) != 0;
}
// gathers bit 7 of the four bytes into a nibble (byte 0 -> bit 0)
__device__ __forceinline__ uint32_t nibble_of(uint32_t hi) {
    return ((((hi >> 7) & 0x01010101u) * 0x00204081u) >> 21) & 0xFu;
}

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
#if defined(__CUDACC__)
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
#else
    return *p;                       // host-run checks of the device code (tests/hostcheck)
#endif
}

__device__ __forceinline__ void append_segment(uint32_t* seg_count, uint32_t* seg_list, int max_segments,
                                               long long seg_global, int seg_per_image, uint32_t mask16) {
    const int img = (int)(seg_global / seg_per_image);
    const uint32_t pos = (uint32_t)(seg_global - (long long)img * seg_per_image);
    const uint32_t slot = atomicAdd(&seg_count[img], 1u);
    if (slot < (uint32_t)max_segments)
        seg_list[(size_t)img * max_segments + slot] = (pos << 16) | mask16;
}

// ---------------------------------------------------------------------------------------------
// sparse per-image reduction
// ---------------------------------------------------------------------------------------------
// NT == 32: the group is one warp (several images per CTA, warp-level synchronisation only);
// NT  > 32: the group is the whole CTA.
template <int NT>
__device__ __forceinline__ void gsync() {
    if (NT == 32) __syncwarp(); else __syncthreads();
}

template <int NT>
__device__ __forceinline__ unsigned block_scan_excl(unsigned v, unsigned& total, unsigned* wsum) {
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned x = v;
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (unsigned)o) x += y;
    }
    if (NT == 32) {
        total = __shfl_sync(0xffffffffu, x, 31);
        return x - v;
    }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    unsigned base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) {
        const unsigned sw = wsum[w];
        if ((unsigned)w < wid) base += sw;
        tot += sw;
    }
    __syncthreads();
    total = tot;
    return base + x - v;
}

// find with path halving: every visited node is re-pointed at its grandparent.  Concurrent writers only
// ever replace a parent by one of its own ancestors, so the forest stays valid without locks.
__device__ __forceinline__ unsigned uf_find(volatile unsigned* parent, unsigned x) {
    unsigned p;
    while ((p = parent[x]) != x) {
        const unsigned gp = parent[p];
        if (gp != p) parent[x] = gp;
        x = gp;
    }
    return x;
}
// lock-free union keeping the smaller index as representative (root == first run in raster order)
__device__ __forceinline__ void uf_unite(unsigned* parent, unsigned a, unsigned b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a < b) { const unsigned tmp = a; a = b; b = tmp; }
        const unsigned old = atomicMin(&parent[a], b);
        if (old == a) return;
        a = old;
    }
}
__device__ __forceinline__ unsigned run_starts(unsigned m) { return m & ~(m << 1) & 0xffffu; }
// sum of the indices of the set bits (branch-free: weight 2^k times the bits whose index has bit k)
__device__ __forceinline__ int bit_index_sum(unsigned m) {
    return __popc(m & 0xAAAAAAAAu) + 2 * __popc(m & 0xCCCCCCCCu) + 4 * __popc(m & 0xF0F0F0F0u) +
           8 * __popc(m & 0xFF00FF00u) + 16 * __popc(m & 0xFFFF0000u);
}
__device__ __forceinline__ int seg_lower_bound(const uint32_t* seg, int n, uint32_t pos) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((seg[mid] >> 16) < pos) lo = mid + 1; else hi = mid;
    }
    return lo;
}

struct BlobSmem;
__device__ __forceinline__ int row_lower_bound(const BlobSmem& sm, int n, int SPR, bool use_table, int rmin, int rmax, uint32_t pos);

struct BlobSmem {
    uint32_t* seg;        // [E]  sorted (pos<<16)|mask
    unsigned* parent;     // [E]  union-find over runs
    uint16_t* base;       // [E]  first run id of segment i
    uint16_t* node_seg;   // [E]
    uint16_t* node_bits;  // [E]
    uint16_t* rank;       // [E]  blob index of a root run
    unsigned long long* acc;   // [MOCAP_ACC_CAP][4]  A2, SX6, SY6, npix
    unsigned* wsum;       // [32]
    uint16_t* rowfirst;   // [row_cap] index of the first segment of row (rmin + k), 0xFFFF = empty; nullptr = binary search
    int row_cap;
    HoleScratch* hs;      // full-size (CTA) reduction only: scratch of the RETR_TREE slow path (blob_holes.cuh); else nullptr
};
// index of the first segment with position >= pos (pos lies in row pos / SPR): through the per-row index
// when the image's rows fit it (one load + a scan over that row's few segments), else by binary search
__device__ __forceinline__ int row_lower_bound(const BlobSmem& sm, int n, int SPR, bool use_table, int rmin, int rmax, uint32_t pos) {
    if (!use_table) return seg_lower_bound(sm.seg, n, pos);
    const int r = (int)(pos / (uint32_t)SPR);
    if (r < rmin || r > rmax) return n;
    int j = sm.rowfirst[r - rmin];
    if (j == 0xFFFF) return n;
    while (j < n && (sm.seg[j] >> 16) < pos) ++j;
    return j;
}

inline size_t blob_reduce_smem_bytes(int E) {
    return (size_t)E * (4 + 4 + 2 + 2 + 2 + 2) + (size_t)MOCAP_ACC_CAP * 32 + 32 * 4 + sizeof(HoleScratch) + 16;
}
__device__ __forceinline__ BlobSmem carve_blob_smem(unsigned char* raw, int E) {
    BlobSmem s;
    s.acc = reinterpret_cast<unsigned long long*>(raw);      raw += (size_t)MOCAP_ACC_CAP * 32;
    s.seg = reinterpret_cast<uint32_t*>(raw);                raw += (size_t)E * 4;
    s.parent = reinterpret_cast<unsigned*>(raw);             raw += (size_t)E * 4;
    s.wsum = reinterpret_cast<unsigned*>(raw);               raw += 32 * 4;
    s.base = reinterpret_cast<uint16_t*>(raw);               raw += (size_t)E * 2;
    s.node_seg = reinterpret_cast<uint16_t*>(raw);           raw += (size_t)E * 2;
    s.node_bits = reinterpret_cast<uint16_t*>(raw);          raw += (size_t)E * 2;
    s.rank = reinterpret_cast<uint16_t*>(raw);                raw += (size_t)E * 2;
    raw += (16 - (reinterpret_cast<uintptr_t>(raw) & 15)) & 15;
    s.hs = reinterpret_cast<HoleScratch*>(raw);
    s.rowfirst = nullptr; s.row_cap = 0;
    return s;
}

// Block-wide: the n segments in sm.seg[0..n) (unsorted) -> blobs of one image.
template <bool WIDE>
__device__ __forceinline__ unsigned long long acc_get(const unsigned long long* acc, unsigned idx) {
    return WIDE ? acc[idx] : (unsigned long long)reinterpret_cast<const unsigned*>(acc)[idx];
}

template <bool WIDE>
__device__ __forceinline__ void acc_add(unsigned long long* acc, unsigned idx, long long v) {
    if (WIDE) acc[idx] += (unsigned long long)v; else reinterpret_cast<unsigned*>(acc)[idx] += (unsigned)v;
}
// Euler number of blob k (kept above the pixel count in accumulator slot 3)
template <bool WIDE>
__device__ __forceinline__ int acc_euler(const unsigned long long* acc, unsigned k) {
    const unsigned long long a3 = acc_get<WIDE>(acc, 4 * k + 3);
    return WIDE ? (int)(long long)(a3 >> 32) : ((int)((unsigned)a3 >> 20) << 20) >> 20;      // sign-extended
}

// RETR_TREE for an image that has a blob with a hole (see blob_holes.cuh).  Whole CTA; runs after the blobs' own
// moments are in sm.acc.  Emits the image's points itself (in cv2's hierarchy order).
template <int NT, bool WIDE>
__device__ __noinline__ void blob_holes_cta(BlobSmem sm, int n, unsigned n_runs, unsigned nb, int W, int H, int max_blobs,
                                            int32_t* __restrict__ out_xy, int32_t* __restrict__ out_n,
                                            int64_t* __restrict__ out_mom, int32_t* __restrict__ out_flags, int flags) {
    const int tid = threadIdx.x % NT;
    const int SPR = W / MOCAP_SEG_PX;
    HoleScratch& hs = *sm.hs;
    // first pixel of every blob (its root run is its first run in raster order)
    for (unsigned id = tid; id < n_runs; id += NT) {
        if (sm.parent[id] != id) continue;
        const unsigned k = sm.rank[id];
        if (k >= nb) continue;
        const uint32_t p = sm.seg[sm.node_seg[id] & 0x7fff] >> 16;
        const int y = p / SPR, sc = p - y * SPR;
        hs.bfirst[k] = (uint32_t)(y * W + 16 * sc + __ffs((int)sm.node_bits[id]) - 1);
        hs.bparent[k] = -1; hs.bbest[k] = 0xffffffffu;
    }
    if (tid == 0) { hs.nholes = 0; hs.unsupported = 0; }
    __syncthreads();
    for (unsigned k = 0; k < nb; ++k) {
        if (acc_euler<WIDE>(sm.acc, k) == 1) continue;               // a solid blob (CTA-uniform)
        if (tid == 0) { hs.bbox[0] = 1 << 30; hs.bbox[1] = 1 << 30; hs.bbox[2] = -1; hs.bbox[3] = -1; }
        __syncthreads();
        for (unsigned id = tid; id < n_runs; id += NT) {
            if (sm.rank[sm.parent[id]] != k) continue;
            const uint32_t p = sm.seg[sm.node_seg[id] & 0x7fff] >> 16;
            const int y = p / SPR, sc = p - y * SPR;
            const unsigned rb = sm.node_bits[id];
            atomicMin(&hs.bbox[0], 16 * sc + __ffs((int)rb) - 1);
            atomicMax(&hs.bbox[2], 16 * sc + 31 - __clz((int)rb));
            atomicMin(&hs.bbox[1], y);
            atomicMax(&hs.bbox[3], y);
        }
        __syncthreads();
        const int x0 = hs.bbox[0], y0 = hs.bbox[1], w = hs.bbox[2] - x0 + 1, h = hs.bbox[3] - y0 + 1;
        if (w + 2 > HOLE_WIN || h + 2 > HOLE_WIN) {                  // does not fit the window: left as the fast path has it
            if (tid == 0) hs.unsupported = 1;
            __syncthreads();
            continue;
        }
        for (int r = tid; r < HOLE_WIN; r += NT) { hs.FS[r] = 0ull; hs.Ex[r] = 0ull; hs.Hm[r] = 0ull; hs.Fh[r] = 0ull; }
        __syncthreads();
        for (unsigned id = tid; id < n_runs; id += NT) {
            if (sm.rank[sm.parent[id]] != k) continue;
            const uint32_t p = sm.seg[sm.node_seg[id] & 0x7fff] >> 16;
            const int y = p / SPR, sc = p - y * SPR;
            const unsigned long long rb = sm.node_bits[id];
            const int sh = 16 * sc + 1 - x0;                         // window bit of the segment's pixel 0
            atomicOr(&hs.FS[y - y0 + 1], sh >= 0 ? (rb << sh) : (rb >> (-sh)));
        }
        __syncthreads();
        if (tid < 32) {                                              // one warp from here; the others wait at the barrier below
            const int lane = tid;
            const unsigned long long Wm = (w + 2 == 64) ? ~0ull : ((1ull << (w + 2)) - 1ull);
            // the complement of the blob inside the window, kept in Ex's place holder Hm while Ex grows
            for (int r = lane; r < HOLE_WIN; r += 32) {
                const unsigned long long fr = r <= h + 1 ? (~hs.FS[r] & Wm) : 0ull;
                hs.Hm[r] = fr;                                                      // "allowed" for the exterior flood
                hs.Ex[r] = (r == 0 || r == h + 1) ? fr : (r <= h ? (fr & (1ull | (1ull << (w + 1)))) : 0ull);
            }
            __syncwarp();
            hole_flood(hs.Ex, hs.Hm, h + 1, lane);
            for (int r = lane; r < HOLE_WIN; r += 32) hs.Hm[r] &= ~hs.Ex[r];         // what the outside does not reach
            __syncwarp();
            const long long sA2 = (long long)acc_get<WIDE>(sm.acc, 4 * k), sSX6 = (long long)acc_get<WIDE>(sm.acc, 4 * k + 1);
            const long long sSY6 = (long long)acc_get<WIDE>(sm.acc, 4 * k + 2);
            long long addA2 = 0, addSX6 = 0, addSY6 = 0;
            while (true) {
                // the first pixel, in raster order, of the regions still to be labelled
                unsigned key = 0xffffffffu;
                for (int r = lane; r <= h; r += 32)
                    if (hs.Hm[r]) { key = min(key, (unsigned)(r * 64 + __ffsll((long long)hs.Hm[r]) - 1)); }
#pragma unroll 1
                for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
                if (key == 0xffffffffu) break;
                const int j = hs.nholes;
                if (j >= HOLE_CAP) { if (lane == 0) hs.unsupported = 1; break; }
                const int r0 = (int)(key >> 6), b0 = (int)(key & 63u);
                for (int r = lane; r < HOLE_WIN; r += 32) hs.Fh[r] = (r == r0) ? (1ull << b0) : 0ull;
                __syncwarp();
                hole_flood(hs.Fh, hs.Hm, h + 1, lane);
                long long size = 0;
                for (int r = lane; r < HOLE_WIN; r += 32) { size += __popcll(hs.Fh[r]); hs.Hm[r] &= ~hs.Fh[r]; }
                size = hole_warp_sum(size);
                long long uA2, uSX6, uSY6;
                hole_cellsum(hs.FS, hs.Fh, h, x0, y0, lane, uA2, uSX6, uSY6);
                const long long hA2 = uA2 - sA2, hSX6 = uSX6 - sSX6, hSY6 = uSY6 - sSY6;
                addA2 += hA2; addSX6 += hSX6; addSY6 += hSY6;
                // blobs whose first pixel lies in this region: the innermost such region is their parent
                for (unsigned t = lane; t < nb; t += 32) {
                    if (t == k) continue;
                    const int ty = (int)(hs.bfirst[t] / (uint32_t)W), tx = (int)(hs.bfirst[t] - (uint32_t)ty * (uint32_t)W);
                    const int wr = ty - y0 + 1, wb = tx - x0 + 1;
                    if (wr >= 0 && wr < HOLE_WIN && wb >= 0 && wb < HOLE_WIN && ((hs.Fh[wr] >> wb) & 1ull) && (uint32_t)size < hs.bbest[t]) {
                        hs.bbest[t] = (uint32_t)size; hs.bparent[t] = (int16_t)j;
                    }
                }
                if (lane == 0) {
                    hs.hA2[j] = hA2; hs.hSX6[j] = hSX6; hs.hSY6[j] = hSY6;
                    hs.hstart[j] = (uint32_t)((y0 - 1 + r0) * W + (x0 - 1 + b0)); hs.hsize[j] = (uint32_t)size; hs.hblob[j] = (uint16_t)k;
                    hs.nholes = j + 1;
                }
                __syncwarp();
            }
            if (lane == 0) {                                         // the blob's outer contour runs around the FILLED blob
                acc_add<WIDE>(sm.acc, 4 * k, addA2); acc_add<WIDE>(sm.acc, 4 * k + 1, addSX6); acc_add<WIDE>(sm.acc, 4 * k + 2, addSY6);
            }
        }
        __syncthreads();
    }
    // emission in cv2's order (one thread: this is the slow path; a few dozen items)
    if (tid == 0) {
        int count = 0;
        if (hs.unsupported) {
            // as the fast path: one centre per blob from its set pixels, reverse raster order.  The blobs handled before
            // the limit was met (and the one at which the hole cap was reached, in part) had their holes' moments added
            // above; every such hole is recorded, so taking them out again restores the set-pixel sums exactly.
            for (int j = 0; j < hs.nholes; ++j) {
                const unsigned b = hs.hblob[j];
                acc_add<WIDE>(sm.acc, 4 * b, -hs.hA2[j]); acc_add<WIDE>(sm.acc, 4 * b + 1, -hs.hSX6[j]);
                acc_add<WIDE>(sm.acc, 4 * b + 2, -hs.hSY6[j]);
            }
            for (int k = (int)nb - 1; k >= 0; --k) {
                const unsigned long long A2 = acc_get<WIDE>(sm.acc, 4 * k);
                if (!A2) continue;
                if (count < max_blobs) {
                    const double m00 = (double)A2 * 0.5, m10 = (double)acc_get<WIDE>(sm.acc, 4 * k + 1) * 0.16666666666666666;
                    const double m01 = (double)acc_get<WIDE>(sm.acc, 4 * k + 2) * 0.16666666666666666;
                    out_xy[2 * count] = (int)(m10 / m00); out_xy[2 * count + 1] = (int)(m01 / m00);
                    if (out_mom) {
                        out_mom[4 * count] = (int64_t)A2; out_mom[4 * count + 1] = (int64_t)acc_get<WIDE>(sm.acc, 4 * k + 1);
                        out_mom[4 * count + 2] = (int64_t)acc_get<WIDE>(sm.acc, 4 * k + 2);
                        out_mom[4 * count + 3] = (int64_t)(acc_get<WIDE>(sm.acc, 4 * k + 3) & (WIDE ? 0xffffffffull : 0xfffffull));
                    }
                }
                ++count;
            }
            flags |= MOCAP_F_HOLES;
        } else {
            // pre-order walk of the hierarchy without recursion: a frame lists either the blobs inside hole `owner`
            // (owner = -1: top level) or the holes of blob `owner`; siblings leave in descending order of their first
            // pixel, found by scanning for the largest key below the one emitted last
            struct Frame { int kind, owner; unsigned long long last; };
            Frame st[34];
            int sp = 0;
            st[0].kind = 0; st[0].owner = -1; st[0].last = ~0ull;
            while (sp >= 0) {
                Frame& f = st[sp];
                int best = -1;
                unsigned long long bkey = 0;
                if (f.kind == 0) {
                    for (int t = 0; t < (int)nb; ++t)
                        if (hs.bparent[t] == f.owner && (unsigned long long)hs.bfirst[t] < f.last && (best < 0 || hs.bfirst[t] > bkey)) { best = t; bkey = hs.bfirst[t]; }
                } else {
                    for (int j = 0; j < hs.nholes; ++j)
                        if (hs.hblob[j] == f.owner && (unsigned long long)hs.hstart[j] < f.last && (best < 0 || hs.hstart[j] > bkey)) { best = j; bkey = hs.hstart[j]; }
                }
                if (best < 0) { --sp; continue; }
                f.last = bkey;
                long long A2, SX6, SY6, npix;
                if (f.kind == 0) {
                    A2 = (long long)acc_get<WIDE>(sm.acc, 4 * best); SX6 = (long long)acc_get<WIDE>(sm.acc, 4 * best + 1);
                    SY6 = (long long)acc_get<WIDE>(sm.acc, 4 * best + 2);
                    npix = (long long)(acc_get<WIDE>(sm.acc, 4 * best + 3) & (WIDE ? 0xffffffffull : 0xfffffull));
                } else { A2 = hs.hA2[best]; SX6 = hs.hSX6[best]; SY6 = hs.hSY6[best]; npix = hs.hsize[best]; }
                if (A2 != 0) {                                       // helpers.py:153: contours of zero area are dropped
                    if (count < max_blobs) {
                        const double m00 = (double)A2 * 0.5, m10 = (double)SX6 * 0.16666666666666666, m01 = (double)SY6 * 0.16666666666666666;
                        out_xy[2 * count] = (int)(m10 / m00); out_xy[2 * count + 1] = (int)(m01 / m00);
                        if (out_mom) { out_mom[4 * count] = A2; out_mom[4 * count + 1] = SX6; out_mom[4 * count + 2] = SY6; out_mom[4 * count + 3] = npix; }
                    }
                    ++count;
                }
                if (sp + 1 < 34) {                                   // descend: a blob's holes, a hole's blobs
                    ++sp;
                    st[sp].kind = f.kind == 0 ? 1 : 0; st[sp].owner = best; st[sp].last = ~0ull;
                }
            }
            flags &= ~MOCAP_F_HOLES;
        }
        if (count > max_blobs) flags |= MOCAP_F_BLOBS;
        *out_n = count < max_blobs ? count : max_blobs;
        if (out_flags) *out_flags = flags;
    }
    __syncthreads();
}

// Returns false (group-uniform) without writing anything when STRICT and a capacity (runs > E,
// blobs > ACC) is exceeded: the caller then hands the image to the full-size kernel.
template <int NT, bool STRICT, bool WIDE>
__device__ __noinline__ bool blob_reduce(BlobSmem sm, int n, int E, int ACC, int W, int H, int max_blobs,
                            int32_t* __restrict__ out_xy, int32_t* __restrict__ out_n,
                            int64_t* __restrict__ out_mom, int32_t* __restrict__ out_flags, int flags_in) {
    const int tid = threadIdx.x % NT;
    const int SPR = W / MOCAP_SEG_PX;     // segments per row
    int flags = flags_in;

    // ---- 1. raster order of (pos<<16 | mask).  Warp groups (n <= 128): rank sort -- every element
    //         counts the smaller ones (keys are unique), no barriers; CTA groups: bitonic sort.
    if (NT == 32 && n <= 40) {
        uint32_t* tmp = reinterpret_cast<uint32_t*>(sm.parent);     // free until step 2
        for (int i = tid; i < n; i += NT) {
            const uint32_t e = sm.seg[i];
            int rank = 0;
            for (int j = 0; j < n; ++j) rank += (sm.seg[j] < e) ? 1 : 0;
            tmp[rank] = e;
        }
        gsync<NT>();
        for (int i = tid; i < n; i += NT) sm.seg[i] = tmp[i];
        gsync<NT>();
    } else if (NT == 32) {
        // stable LSD radix sort of the 16-bit positions, 8 bits per pass; histogram in the (not yet used)
        // accumulator slab, ping-pong between seg[] and the parent[] array
        uint32_t* hist = reinterpret_cast<uint32_t*>(sm.acc);       // [256]
        uint32_t* src = sm.seg;
        uint32_t* dst = reinterpret_cast<uint32_t*>(sm.parent);
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            const int shift = 16 + 8 * pass;
            for (int k = tid; k < 256; k += 32) hist[k] = 0u;
            gsync<NT>();
            for (int i = tid; i < n; i += 32) atomicAdd(&hist[(src[i] >> shift) & 0xffu], 1u);
            gsync<NT>();
            {   // exclusive scan of the 256 bins: 8 consecutive bins per lane
                unsigned loc[8], sum = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) { loc[k] = hist[tid * 8 + k]; sum += loc[k]; }
                unsigned tot;
                unsigned run = block_scan_excl<NT>(sum, tot, sm.wsum);
#pragma unroll
                for (int k = 0; k < 8; ++k) { hist[tid * 8 + k] = run; run += loc[k]; }
            }
            gsync<NT>();
            for (int i0 = 0; i0 < n; i0 += 32) {                    // stable scatter, 32 elements at a time
                const int i = i0 + tid;
                const bool act = i < n;
                const uint32_t e = act ? src[i] : 0u;
                const unsigned d = act ? ((e >> shift) & 0xffu) : 0x100u + tid;     // inactive lanes: unique keys
                const unsigned peers = __match_any_sync(0xffffffffu, d);
                const unsigned below = __popc(peers & ((1u << tid) - 1u));
                unsigned base_pos = 0;
                if (act) base_pos = hist[d];
                __syncwarp();
                if (act && below == 0) hist[d] = base_pos + __popc(peers);
                if (act) dst[base_pos + below] = e;
                __syncwarp();
            }
            uint32_t* t2 = src; src = dst; dst = t2;
        }
        // two passes: the result is back in seg[]
        gsync<NT>();
    } else {
        int n2 = 1;
        while (n2 < n) n2 <<= 1;
        for (int i = n + tid; i < n2; i += NT) sm.seg[i] = SEG_PAD;
        gsync<NT>();
        for (int k = 2; k <= n2; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = tid; i < n2; i += NT) {
                    const int ixj = i ^ j;
                    if (ixj > i) {
                        const uint32_t a = sm.seg[i], b = sm.seg[ixj];
                        const bool up = ((i & k) == 0);
                        if ((a > b) == up) { sm.seg[i] = b; sm.seg[ixj] = a; }
                    }
                }
                gsync<NT>();
            }
        }
    }

    // per-row index of the sorted list (neighbour rows are looked up many times per run)
    const int rmin = (int)((sm.seg[0] >> 16) / (uint32_t)SPR), rmax = (int)((sm.seg[n - 1] >> 16) / (uint32_t)SPR);
    const bool use_table = sm.rowfirst != nullptr && (rmax - rmin) < sm.row_cap;
    if (use_table) {
        for (int k = tid; k <= rmax - rmin; k += NT) sm.rowfirst[k] = 0xFFFFu;
        gsync<NT>();
        for (int i = tid; i < n; i += NT) {
            const int r = (int)((sm.seg[i] >> 16) / (uint32_t)SPR);
            if (i == 0 || (int)((sm.seg[i - 1] >> 16) / (uint32_t)SPR) != r) sm.rowfirst[r - rmin] = (uint16_t)i;
        }
        gsync<NT>();
    }

    // ---- 2. runs (maximal horizontal strings of set pixels inside one 16-px segment) become nodes
    unsigned n_runs = 0;
    {
        unsigned carry = 0;
        for (int i0 = 0; i0 < n; i0 += NT) {
            const int i = i0 + tid;
            const unsigned cnt = (i < n) ? __popc(run_starts(sm.seg[i] & 0xffffu)) : 0u;
            unsigned tot;
            const unsigned ex = block_scan_excl<NT>(cnt, tot, sm.wsum);
            if (i < n) sm.base[i] = (uint16_t)min(carry + ex, 0xffffu);
            carry += tot;
        }
        n_runs = carry;
    }
    if (n_runs > (unsigned)E) {          // cannot label: report and emit nothing (group-uniform)
        if (STRICT) return false;
        if (tid == 0) { *out_n = 0; if (out_flags) *out_flags = flags | MOCAP_F_SEGMENTS; }
        return true;
    }
    for (int i = tid; i < n; i += NT) {
        unsigned s = sm.seg[i] & 0xffffu;
        unsigned id = sm.base[i];
        while (s) {
            const unsigned b = s & (0u - s);
            const unsigned run = s & ~(s + b);
            s &= ~run;
            sm.node_seg[id] = (uint16_t)i;
            sm.node_bits[id] = (uint16_t)run;
            sm.parent[id] = id;
            ++id;
        }
    }
    gsync<NT>();

    // ---- 3. 8-connectivity unions: right neighbour across the segment boundary, and the row above
    for (unsigned id = tid; id < n_runs; id += NT) {
        const int i = sm.node_seg[id];
        const unsigned rb = sm.node_bits[id];
        const uint32_t p = sm.seg[i] >> 16;
        const int y = p / SPR, sc = p - y * SPR;
        if ((rb & 0x8000u) && sc + 1 < SPR && i + 1 < n) {
            const uint32_t e2 = sm.seg[i + 1];
            if ((e2 >> 16) == p + 1 && (e2 & 1u)) uf_unite(sm.parent, id, sm.base[i + 1]);
        }
        unsigned U = 0;                                            // 18-bit window of row y-1 over columns 16*sc-1 .. 16*sc+16
        if (y > 0) {                                               // the <= 3 segments of row y-1 that touch this run
            const unsigned ext = (rb | (rb << 1) | (rb >> 1)) & 0xffffu;
            const uint32_t q = p - SPR;
            const int lo = row_lower_bound(sm, n, SPR, use_table, rmin, rmax, sc > 0 ? q - 1 : q);
            for (int j = lo; j < n && j < lo + 3; ++j) {
                const uint32_t ej = sm.seg[j], pj = ej >> 16;
                if (pj > q + 1) break;
                const unsigned mm = ej & 0xffffu;
                if (pj == q) U |= mm << 1;
                else if (pj + 1 == q) U |= (mm >> 15) & 1u;
                else if (sc + 1 < SPR) U |= (mm & 1u) << 17;
                if (pj == q) {
                    unsigned sbits = mm, r = 0;
                    while (sbits) {
                        const unsigned b = sbits & (0u - sbits);
                        const unsigned run = sbits & ~(sbits + b);
                        sbits &= ~run;
                        if (run & ext) uf_unite(sm.parent, id, sm.base[j] + r);
                        ++r;
                    }
                } else if (pj + 1 == q) {                           // left neighbour segment (only searched when sc > 0)
                    if ((rb & 1u) && (mm & 0x8000u)) uf_unite(sm.parent, id, sm.base[j] + __popc(run_starts(mm)) - 1);
                } else if (sc + 1 < SPR) {                          // pj == q + 1: right neighbour segment
                    if ((rb & 0x8000u) && (mm & 1u)) uf_unite(sm.parent, id, sm.base[j]);
                }
            }
        }
        // Euler number, part 1 (see step 5): the run's first pixel opens a new run of (row y-1 | row y) that
        // row y-1 does not own -- neither the pixel above it nor the one above-left is set (above-left-of-left is
        // decided in step 5 together with this row's own left neighbour).  Kept in bit 15 of node_seg (< 4096).
        {
            const int s0 = __ffs((int)rb);                          // window index of the run's first pixel (bit + 1)
            if (!((U >> s0) & 1u) && !((U >> (s0 - 1)) & 1u)) sm.node_seg[id] |= 0x8000u;
        }
    }
    gsync<NT>();
    // flatten (two phases so that nobody chases a pointer that is being rewritten;
    // sm.rank is free until step 4 and run ids fit 16 bits because n_runs <= E <= 4096)
    for (unsigned id = tid; id < n_runs; id += NT) sm.rank[id] = (uint16_t)uf_find(sm.parent, id);
    gsync<NT>();
    for (unsigned id = tid; id < n_runs; id += NT) sm.parent[id] = sm.rank[id];
    gsync<NT>();

    // ---- 4. rank the roots (ascending run id == ascending raster position of the blob's first pixel)
    unsigned n_blobs = 0;
    {
        unsigned carry = 0;
        for (unsigned i0 = 0; i0 < n_runs; i0 += NT) {
            const unsigned id = i0 + tid;
            const unsigned is_root = (id < n_runs && sm.parent[id] == id) ? 1u : 0u;
            unsigned tot;
            const unsigned ex = block_scan_excl<NT>(is_root, tot, sm.wsum);
            if (is_root) sm.rank[id] = (uint16_t)min(carry + ex, 0xffffu);
            carry += tot;
        }
        n_blobs = carry;
    }
    if (n_blobs > (unsigned)ACC) {
        if (STRICT) return false;
        flags |= MOCAP_F_BLOBS;
    }
    const unsigned nb = min(n_blobs, (unsigned)ACC);
    for (unsigned k = tid; k < nb * 4; k += NT) { if (WIDE) sm.acc[k] = 0ull; else reinterpret_cast<unsigned*>(sm.acc)[k] = 0u; }
    gsync<NT>();

    // ---- 5. per-run share of the 2x2-cell moments.  A cell is owned by the run holding its
    //         top-left corner, or its top-right corner when the top-left pixel is clear.
    for (unsigned id = tid; id < n_runs; id += NT) {
        const unsigned blob = sm.rank[sm.parent[id]];
        if (blob >= (unsigned)ACC) continue;
        const int i = sm.node_seg[id] & 0x7fff;
        const unsigned up_open = sm.node_seg[id] >> 15;
        const unsigned rb = sm.node_bits[id];
        const uint32_t e = sm.seg[i];
        const uint32_t p = e >> 16;
        const unsigned m = e & 0xffffu;
        const int y = p / SPR, sc = p - y * SPR;
        // 18-bit windows over columns 16*sc-1 .. 16*sc+16 of rows y (T) and y+1 (Bw)
        unsigned T = m << 1;
        if (sc > 0 && i > 0 && (sm.seg[i - 1] >> 16) == p - 1) T |= (sm.seg[i - 1] >> 15) & 1u;
        if (sc + 1 < SPR && i + 1 < n && (sm.seg[i + 1] >> 16) == p + 1) T |= (sm.seg[i + 1] & 1u) << 17;
        unsigned Bw = 0;
        if (y + 1 < H) {
            const uint32_t q = p + SPR;
            const int lo = row_lower_bound(sm, n, SPR, use_table, rmin, rmax, sc > 0 ? q - 1 : q);
            for (int j = lo; j < n && j < lo + 3; ++j) {
                const uint32_t ej = sm.seg[j], pj = ej >> 16;
                if (pj > q + 1) break;
                if (pj == q) Bw |= (ej & 0xffffu) << 1;
                else if (pj + 1 == q) Bw |= (ej >> 15) & 1u;        // only searched when sc > 0
                else if (sc + 1 < SPR) Bw |= (ej & 1u) << 17;
            }
        }
        const unsigned Rw = rb << 1;
        const unsigned T1 = T >> 1, B1 = Bw >> 1;
        const unsigned own = (Rw | (~T & (Rw >> 1))) & 0x1ffffu;
        const unsigned full = T & T1 & Bw & B1 & own;
        const unsigned mtl = ~T & T1 & Bw & B1 & own;      // triangle, top-left corner missing
        const unsigned mtr = T & ~T1 & Bw & B1 & own;
        const unsigned mbl = T & T1 & ~Bw & B1 & own;
        const unsigned mbr = T & T1 & Bw & ~B1 & own;
        const int nf = __popc(full), ntl = __popc(mtl), ntr = __popc(mtr), nbl = __popc(mbl), nbr = __popc(mbr);
        const long long x0 = 16ll * sc - 1;               // column of window bit 0
        const long long sxf = x0 * nf + bit_index_sum(full);
        const long long sx_tl = x0 * ntl + bit_index_sum(mtl), sx_tr = x0 * ntr + bit_index_sum(mtr);
        const long long sx_bl = x0 * nbl + bit_index_sum(mbl), sx_br = x0 * nbr + bit_index_sum(mbr);
        const long long a2 = 2ll * nf + ntl + ntr + nbl + nbr;
        const long long sx6 = 6 * sxf + 3ll * nf + 3 * (sx_tl + sx_tr + sx_bl + sx_br) + 2ll * (ntl + nbl) + (ntr + nbr);
        const long long sy6 = (6ll * y + 3) * nf + (3ll * y + 2) * (ntl + ntr) + (3ll * y + 1) * (nbl + nbr);
        // Euler number of the blob (components - holes, 8-connectivity) from runs: sum over rows of the runs of
        // (row y-1 | row y), minus the runs of every row (two rows whose runs touch merge into one run of the OR, and
        // the touching graph between two rows is a forest).  Each run of an OR is counted at its first pixel, by the
        // run that holds it; only a run that is not the continuation of a run of the left segment can start one.
        int euler = 0;
        {
            const int s0 = __ffs((int)rb);                          // window index of the run's first pixel
            if (!((T >> (s0 - 1)) & 1u))                            // a true run start: -1 for the row's own run count,
                euler = (int)(!((Bw >> (s0 - 1)) & 1u)) + (int)(up_open && true) - 1;   // +1 per OR-run it opens (below / above)
        }
        if (WIDE) {
            unsigned long long* a = sm.acc + 4 * blob;
            if (a2) {
                atomicAdd(a + 0, (unsigned long long)a2);
                atomicAdd(a + 1, (unsigned long long)sx6);
                atomicAdd(a + 2, (unsigned long long)sy6);
            }
            atomicAdd(a + 3, (unsigned long long)__popc(rb) + ((unsigned long long)(long long)euler << 32));
        } else {                                                   // 6*max(W,H)*W*H < 2^32: native 32-bit shared atomics
            unsigned* a = reinterpret_cast<unsigned*>(sm.acc) + 4 * blob;
            if (a2) {
                atomicAdd(a + 0, (unsigned)a2);
                atomicAdd(a + 1, (unsigned)sx6);
                atomicAdd(a + 2, (unsigned)sy6);
            }
            atomicAdd(a + 3, (unsigned)__popc(rb) + ((unsigned)euler << 20));       // pixel count < 2^20, Euler number mod 4096 above it
        }
    }
    gsync<NT>();

    // ---- 6. keep blobs with non-zero polygon area (helpers.py:153), emit in reverse raster order
    unsigned n_keep = 0;
    {
        unsigned carry = 0, holed = 0;
        for (unsigned k0 = 0; k0 < nb; k0 += NT) {      // pass 1: count; a blob's Euler number is 1 - (number of holes)
            const unsigned k = k0 + tid;
            const unsigned keep = (k < nb && acc_get<WIDE>(sm.acc, 4 * k) != 0ull) ? 1u : 0u;
            unsigned has_hole = 0;
            if (k < nb) {
                const unsigned long long a3 = acc_get<WIDE>(sm.acc, 4 * k + 3);
                const int eu = WIDE ? (int)(long long)(a3 >> 32) : ((int)((unsigned)a3 >> 20) << 20) >> 20;      // sign-extended
                has_hole = eu != 1 ? 1u : 0u;
            }
            unsigned tot;
            block_scan_excl<NT>(keep | (has_hole << 16), tot, sm.wsum);
            carry += tot & 0xffffu;
            holed += tot >> 16;
        }
        // cv.findContours(RETR_TREE) gives every hole a contour of its own (one more point, helpers.py:147-158) and
        // the outer contour's moments are those of the FILLED blob: this path reports the set pixels' polygon and
        // says so
        if (holed) {
            if (STRICT) return false;                    // the one-warp path hands the image to the full-size reduction
            if (NT > 32 && sm.hs != nullptr) {           // RETR_TREE slow path (blob_holes.cuh); it emits the image itself
                blob_holes_cta<NT, WIDE>(sm, n, n_runs, nb, W, H, max_blobs, out_xy, out_n, out_mom, out_flags, flags);
                return true;
            }
            flags |= MOCAP_F_HOLES;
        }
        n_keep = carry;
        carry = 0;
        for (unsigned k0 = 0; k0 < nb; k0 += NT) {      // pass 2: place
            const unsigned k = k0 + tid;
            const unsigned keep = (k < nb && acc_get<WIDE>(sm.acc, 4 * k) != 0ull) ? 1u : 0u;
            unsigned tot;
            const unsigned ex = block_scan_excl<NT>(keep, tot, sm.wsum);
            if (keep) {
                const unsigned o = n_keep - 1 - (carry + ex);
                if (o < (unsigned)max_blobs) {
                    const unsigned long long A2 = acc_get<WIDE>(sm.acc, 4 * k), SX6 = acc_get<WIDE>(sm.acc, 4 * k + 1), SY6 = acc_get<WIDE>(sm.acc, 4 * k + 2);
                    const double m00 = (double)A2 * 0.5;                       // cv.moments: a00 * 0.5
                    const double m10 = (double)SX6 * 0.16666666666666666;      //             a10 * (1/6)
                    const double m01 = (double)SY6 * 0.16666666666666666;
                    out_xy[2 * o + 0] = (int)(m10 / m00);                       // int(m10/m00), helpers.py:154
                    out_xy[2 * o + 1] = (int)(m01 / m00);
                    if (out_mom) {
                        out_mom[4 * o + 0] = (int64_t)A2; out_mom[4 * o + 1] = (int64_t)SX6;
                        out_mom[4 * o + 2] = (int64_t)SY6;
                        out_mom[4 * o + 3] = (int64_t)(acc_get<WIDE>(sm.acc, 4 * k + 3) & (WIDE ? 0xffffffffull : 0xfffffull));
                    }
                }
            }
            carry += tot;
        }
    }
    if (tid == 0) {
        if (n_keep > (unsigned)max_blobs) flags |= MOCAP_F_BLOBS;
        *out_n = (int)min(n_keep, (unsigned)max_blobs);
        if (out_flags) *out_flags = flags;
    }
    return true;
}

#define BLOB_WE   256     // segments (and runs) a warp handles
#define BLOB_WACC 64      // blobs a warp accumulates
#define BLOB_ROWS 512     // image rows the per-warp row index spans (larger spans fall back to binary search)
struct WarpSlab {
    unsigned long long acc[BLOB_WACC * 4];
    uint32_t seg[BLOB_WE];
    unsigned parent[BLOB_WE];
    uint16_t base[BLOB_WE], node_seg[BLOB_WE], node_bits[BLOB_WE], rank[BLOB_WE];
};
// The per-row index lives in the upper half of acc[] when the accumulators are 32-bit (they then need
// only 1 KB of the 2 KB); with 64-bit accumulators the lookup falls back to binary search.
#define BLOB_ROWFIRST(sl, WIDE) ((WIDE) ? (uint16_t*)nullptr : reinterpret_cast<uint16_t*>(reinterpret_cast<unsigned char*>((sl).acc) + BLOB_WACC * 16))

