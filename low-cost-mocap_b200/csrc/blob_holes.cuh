// S1, blobs WITH holes: what cv.findContours(RETR_TREE) + cv.moments make of them (reference
// computer_code/api/helpers.py:147-158), for the rare images the fast path flags.
//
// RETR_TREE gives every hole a contour of its own, and the outer contour of a blob is traced around the blob with its
// holes FILLED.  In the 2x2-cell formulation of blob_device.cuh (cellsum(M) = the integers A2, SX6, SY6 of the polygon
// through the pixel centres of the solid set M) this is, for a blob S and a hole whose enclosed region is `fill`
// (a 4-connected component of the complement of S that does not reach the outside -- it contains the hole's
// background pixels AND whatever lies inside the hole, nested blobs included):
//      moments of the hole contour          = cellsum(S | fill) - cellsum(S)
//      moments of the blob's outer contour  = cellsum(S) + sum over its holes of the above
// and the contours leave in the order cv2 walks its hierarchy: top-level blobs in descending raster order of
// their first pixel; after a blob its holes in descending raster order of their first pixel; after a hole the blobs
// that sit directly inside it, same rule, recursively.  Checked against cv2 on random images (rings, nested rings,
// porous patches, blobs inside holes): tests/test_device_code_on_host.py, tests/test_parity_gpu.py.
//
// This is the slow path: it runs in the full-size (one CTA per image) reduction only -- the one-warp-per-image fast
// path hands images whose Euler numbers show a hole to the worklist -- on a 64 x 64 bitmap window per holed blob.
// A holed blob wider or taller than 62 pixels, or more than HOLE_CAP holes in one image, makes the whole image leave as
// the fast path computes it (one centre per blob from its set pixels: the hole moments already added are taken out
// again) and the image keeps MOCAP_F_HOLES; otherwise the bit is cleared: the result is the reference's.
//
// Opt-in (mocap_set_large_holes): a holed blob that does not fit the 64 x 64 window is handled in a whole-image window
// instead, four bitmaps of (h + 2) rows x ceil((w + 2) / 64) 64-bit words per CTA in global memory, worked on by the
// whole CTA (blob_holes_wide in blob_device.cuh).  Then only more than HOLE_CAP holes leave the bit.
#pragma once
#include "common.cuh"

#define HOLE_WIN 64
#define HOLE_CAP 64

struct HoleScratch {
    unsigned long long FS[HOLE_WIN];      // the blob, one bit per pixel, window = bounding box + 1 px margin
    unsigned long long Ex[HOLE_WIN];      // complement reached from the margin
    unsigned long long Hm[HOLE_WIN];      // complement NOT reached: the holes' enclosed regions still to be labelled
    unsigned long long Fh[HOLE_WIN];      // the region of the hole at hand
    long long hA2[HOLE_CAP], hSX6[HOLE_CAP], hSY6[HOLE_CAP];
    uint32_t hstart[HOLE_CAP], hsize[HOLE_CAP];
    uint16_t hblob[HOLE_CAP];
    uint32_t bfirst[MOCAP_ACC_CAP];       // raster position of every blob's first pixel
    uint32_t bbest[MOCAP_ACC_CAP];        // size of the innermost hole region found so far that contains it
    int16_t bparent[MOCAP_ACC_CAP];       // that hole, -1: top level
    int bbox[4];
    int nholes, unsupported;
};

__device__ __forceinline__ long long hole_warp_sum(long long v) {
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ long long bit_index_sum64(unsigned long long m) {
    long long s = 0;
    s += __popcll(m & 0xAAAAAAAAAAAAAAAAull);
    s += 2ll * __popcll(m & 0xCCCCCCCCCCCCCCCCull);
    s += 4ll * __popcll(m & 0xF0F0F0F0F0F0F0F0ull);
    s += 8ll * __popcll(m & 0xFF00FF00FF00FF00ull);
    s += 16ll * __popcll(m & 0xFFFF0000FFFF0000ull);
    s += 32ll * __popcll(m & 0xFFFFFFFF00000000ull);
    return s;
}

// 4-neighbour flood inside `allowed` from the seeds in `grow` (both [HOLE_WIN] in shared memory), rows 1 .. last:
// one warp, every lane owns rows lane and lane + 32; repeated until no row changes
__device__ __forceinline__ void hole_flood(unsigned long long* grow, const unsigned long long* allowed, int last, int lane) {
    while (true) {
        bool changed = false;
        for (int r = lane; r <= last; r += 32) {
            if (r == 0) continue;
            const unsigned long long g = grow[r];
            const unsigned long long up = grow[r - 1], dn = r + 1 < HOLE_WIN ? grow[r + 1] : 0ull;
            unsigned long long ng = g | (allowed[r] & ((g << 1) | (g >> 1) | up | dn));
            // run the row to its ends at once: a seed fills the whole stretch of allowed pixels it sits in
            unsigned long long prev;
            do { prev = ng; ng |= allowed[r] & ((ng << 1) | (ng >> 1)); } while (ng != prev);
            if (ng != g) { grow[r] = ng; changed = true; }
        }
        __syncwarp();
        if (!__ballot_sync(0xffffffffu, changed ? 1 : 0)) break;
    }
}

// cellsum of the window bitmap U (rows 0 .. h + 1), in IMAGE coordinates (window bit b of row r = pixel (x0 - 1 + b, y0 - 1 + r))
__device__ __forceinline__ void hole_cellsum(const unsigned long long* FS, const unsigned long long* Fh, int h, int x0, int y0, int lane,
                                             long long& A2, long long& SX6, long long& SY6) {
    long long a2 = 0, sx6 = 0, sy6 = 0;
    for (int r = lane; r <= h; r += 32) {                           // cells between rows r and r + 1
        const unsigned long long T = FS[r] | Fh[r], B = FS[r + 1] | Fh[r + 1];
        const unsigned long long T1 = T >> 1, B1 = B >> 1;
        const unsigned long long full = T & T1 & B & B1;
        const unsigned long long mtl = ~T & T1 & B & B1, mtr = T & ~T1 & B & B1, mbl = T & T1 & ~B & B1, mbr = T & T1 & B & ~B1;
        const long long nf = __popcll(full), ntl = __popcll(mtl), ntr = __popcll(mtr), nbl = __popcll(mbl), nbr = __popcll(mbr);
        const long long sxf = bit_index_sum64(full);
        const long long sxt = bit_index_sum64(mtl) + bit_index_sum64(mtr) + bit_index_sum64(mbl) + bit_index_sum64(mbr);
        a2 += 2 * nf + ntl + ntr + nbl + nbr;
        sx6 += 6 * sxf + 3 * nf + 3 * sxt + 2 * (ntl + nbl) + (ntr + nbr);
        sy6 += (6ll * r + 3) * nf + (3ll * r + 2) * (ntl + ntr) + (3ll * r + 1) * (nbl + nbr);
    }
    a2 = hole_warp_sum(a2); sx6 = hole_warp_sum(sx6); sy6 = hole_warp_sum(sy6);
    A2 = a2;
    SX6 = sx6 + 3ll * (x0 - 1) * a2;                                // a full cell moves by 6 d = 3 d * 2, a triangle by 3 d * 1
    SY6 = sy6 + 3ll * (y0 - 1) * a2;
}

// ---- whole-image window (opt-in).  A bitmap holds rows 0 .. h + 1 of nw words each, row r word q at r * nw + q; bit b
// of word q in row r is pixel (x0 - 1 + 64 q + b, y0 - 1 + r).  Scratch of one CTA: four bitmaps of hole_wide_words.
inline __host__ __device__ size_t hole_wide_words(int W, int H) { return (size_t)(H + 2) * (size_t)((W + 2 + 63) / 64); }

// occluded fills inside one word (Kogge-Stone): the seeds g grown through the allowed bits p towards higher / lower bits
__device__ __forceinline__ unsigned long long fill_up64(unsigned long long g, unsigned long long p) {
    g &= p;
    g |= p & (g << 1);  p &= p << 1;
    g |= p & (g << 2);  p &= p << 2;
    g |= p & (g << 4);  p &= p << 4;
    g |= p & (g << 8);  p &= p << 8;
    g |= p & (g << 16); p &= p << 16;
    g |= p & (g << 32);
    return g;
}
__device__ __forceinline__ unsigned long long fill_down64(unsigned long long g, unsigned long long p) {
    g &= p;
    g |= p & (g >> 1);  p &= p >> 1;
    g |= p & (g >> 2);  p &= p >> 2;
    g |= p & (g >> 4);  p &= p >> 4;
    g |= p & (g >> 8);  p &= p >> 8;
    g |= p & (g >> 16); p &= p >> 16;
    g |= p & (g >> 32);
    return g;
}

// one row of the flood: the allowed pixels under / over a grown pixel of rows r - 1, r + 1 join, then every stretch of
// allowed pixels that holds a grown one fills, across word boundaries (a sweep up the words, then one down).  Only row r
// is written.  Returns whether it grew.
__device__ __forceinline__ bool hole_wide_row(unsigned long long* g, const unsigned long long* a, int nw, int r) {
    unsigned long long* gr = g + (size_t)r * nw;
    const unsigned long long* ar = a + (size_t)r * nw;
    const unsigned long long *up = gr - nw, *dn = gr + nw;
    bool grew = false;
    unsigned long long carry = 0;
    for (int q = 0; q < nw; ++q) {
        const unsigned long long old = gr[q], al = ar[q];
        const unsigned long long v = fill_up64(old | (al & (up[q] | dn[q] | carry)), al);
        carry = v >> 63;                                            // bit 0 of the next word
        if (v != old) { gr[q] = v; grew = true; }
    }
    carry = 0;
    for (int q = nw - 1; q >= 0; --q) {
        const unsigned long long old = gr[q], al = ar[q];
        const unsigned long long v = fill_down64(old | (al & (carry << 63)), al);
        carry = v & 1ull;                                           // bit 63 of the word below
        if (v != old) { gr[q] = v; grew = true; }
    }
    return grew;
}

// 4-neighbour flood inside `allowed` from the seeds in `grow`, rows 1 .. h, whole CTA.  Thread t owns a band of rows
// and sweeps it down and up; even and odd bands take turns, so a band only reads its neighbours' edge rows while they
// stand still.  Repeated until a round changes nothing: the set only grows, so it ends.  flag: two words of shared memory.
template <int NT>
__device__ __forceinline__ void hole_wide_flood(unsigned long long* grow, const unsigned long long* allowed, int nw, int h, int tid,
                                                unsigned* flag) {
    const int band = (h + NT - 1) / NT, lo = 1 + tid * band, hi = min(h, lo + band - 1);
    int s = 0;
    if (tid == 0) flag[0] = 0u;
    while (true) {
        bool grew = false;
        for (int parity = 0; parity < 2; ++parity) {
            if ((tid & 1) == parity) {
                for (int r = lo; r <= hi; ++r) grew |= hole_wide_row(grow, allowed, nw, r);
                for (int r = hi - 1; r >= lo; --r) grew |= hole_wide_row(grow, allowed, nw, r);
            }
            if (parity == 0) {
                __syncthreads();
                if (tid == 0) flag[s ^ 1] = 0u;                     // last read before this barrier; next written after the one below
            }
        }
        if (grew) atomicOr(&flag[s], 1u);
        __syncthreads();
        const unsigned any = flag[s];
        s ^= 1;
        if (!any) return;
    }
}

// CTA-wide minimum / sums through shared slots (three barriers: the slots are free again when it returns)
template <int NT>
__device__ __forceinline__ unsigned cta_min_u32(unsigned v, unsigned* slot, int tid) {
    if (tid == 0) *slot = 0xffffffffu;
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((tid & 31) == 0) atomicMin(slot, v);
    __syncthreads();
    v = *slot;
    __syncthreads();
    return v;
}
template <int NT>
__device__ __forceinline__ void cta_sum4(long long* v, unsigned long long* slot, int tid) {
    if (tid < 4) slot[tid] = 0ull;
    for (int i = 0; i < 4; ++i) v[i] = hole_warp_sum(v[i]);
    __syncthreads();
    if ((tid & 31) == 0)
        for (int i = 0; i < 4; ++i) atomicAdd(&slot[i], (unsigned long long)v[i]);
    __syncthreads();
    for (int i = 0; i < 4; ++i) v[i] = (long long)slot[i];
    __syncthreads();
}

// this thread's share of the cellsum of FS | Fh in the whole-image window, in WINDOW coordinates (cells between rows r, r + 1)
template <int NT>
__device__ __forceinline__ void hole_wide_cellsum(const unsigned long long* FS, const unsigned long long* Fh, int nw, int h, int tid,
                                                  long long& A2, long long& SX6, long long& SY6) {
    long long a2 = 0, sx6 = 0, sy6 = 0;
    for (int r = tid; r <= h; r += NT) {
        const size_t t0 = (size_t)r * nw, b0 = t0 + nw;
        for (int q = 0; q < nw; ++q) {
            const unsigned long long T = FS[t0 + q] | Fh[t0 + q], B = FS[b0 + q] | Fh[b0 + q];
            const unsigned long long Tn = q + 1 < nw ? (FS[t0 + q + 1] | Fh[t0 + q + 1]) : 0ull;
            const unsigned long long Bn = q + 1 < nw ? (FS[b0 + q + 1] | Fh[b0 + q + 1]) : 0ull;
            const unsigned long long T1 = (T >> 1) | (Tn << 63), B1 = (B >> 1) | (Bn << 63);
            const unsigned long long full = T & T1 & B & B1;
            const unsigned long long mtl = ~T & T1 & B & B1, mtr = T & ~T1 & B & B1, mbl = T & T1 & ~B & B1, mbr = T & T1 & B & ~B1;
            const long long nf = __popcll(full), ntl = __popcll(mtl), ntr = __popcll(mtr), nbl = __popcll(mbl), nbr = __popcll(mbr);
            const long long xq = 64ll * q;
            const long long sxf = bit_index_sum64(full) + xq * nf;
            const long long sxt = bit_index_sum64(mtl) + bit_index_sum64(mtr) + bit_index_sum64(mbl) + bit_index_sum64(mbr) +
                                  xq * (ntl + ntr + nbl + nbr);
            a2 += 2 * nf + ntl + ntr + nbl + nbr;
            sx6 += 6 * sxf + 3 * nf + 3 * sxt + 2 * (ntl + nbl) + (ntr + nbr);
            sy6 += (6ll * r + 3) * nf + (3ll * r + 2) * (ntl + ntr) + (3ll * r + 1) * (nbl + nbr);
        }
    }
    A2 = a2; SX6 = sx6; SY6 = sy6;
}
