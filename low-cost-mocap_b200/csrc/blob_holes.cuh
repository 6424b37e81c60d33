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
