// Marker triplets -> drone records for ONE frame-set: the body of k_locate_objects (locate_kernels.cu).  Written against
// geom.cuh only (no CUDA headers), so that tests/hostcheck/locate_host.cpp runs this very code with g++ and the kernel
// runs it with one thread per frame-set.
//
// Replaces locate_objects (reference computer_code/api/helpers.py:424-480): pairwise distance matrix of
// the frame's 3D points; a point i with >= 2 neighbours at 0.095 +- 0.025 looks, in the reference's
// cartesian-product order, for the first ordered pair (a, b) of those neighbours that is 0.15 +- 0.025
// apart; the object sits midway between a and b, heads along a - b (folded into [-pi/2, pi/2], sign
// flipped), its error is the mean of the three reprojection errors and its droneIndex comes from the
// side of the axis point i lies on.  i, a and b all go on the reference's already_matched_points list, but that list
// only screens the OUTER index: a matched point is skipped as a later i, yet stays available as a / b of another
// i (so up to one object per point can come out; the mirror sizes max_objects accordingly).
// The two tolerance tests are not alike: a neighbour needs |d - 0.095| < 0.025, a pair is refused on
// |d - 0.15| > 0.025 (so equality passes).  Every comparison is false on NaN, as numpy's are.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "geom.cuh"

#define LOC_D1 0.095
#define LOC_D2 0.15
#define LOC_TOL 0.025
#define LOC_MAX_POINTS 128      // the matched-points set is two 64-bit words

GEOM_HD double pt_dist(const double* __restrict__ P, int a, int b) {
    const double dx = DSUB(P[3 * a], P[3 * b]), dy = DSUB(P[3 * a + 1], P[3 * b + 1]), dz = DSUB(P[3 * a + 2], P[3 * b + 2]);
    return sqrt(DADD(DADD(DMUL(dx, dx), DMUL(dy, dy)), DMUL(dz, dz)));      // np.sqrt(np.sum((a-b)**2)), helpers.py:434,446
}

// The greedy scan of one frame-set: P [K][3], E [K].  Writes the first max_objects records to out [max_objects][5] =
// {x, y, z, heading, error} and drone_index [max_objects]; returns the number FOUND, which may exceed max_objects.
GEOM_HD int locate_scan(const double* __restrict__ P, const double* __restrict__ E, int K, int max_objects,
                        double* __restrict__ out, int32_t* __restrict__ drone_index) {
    // bit i of used: point i already produced an object (helpers.py:436-437)
    unsigned long long used_lo = 0ull, used_hi = 0ull;
    int found = 0;
    for (int i = 0; i < K; ++i) {
        if ((i < 64 ? (used_lo >> i) : (used_hi >> (i - 64))) & 1ull) continue;
        int cnt = 0;
        for (int j = 0; j < K; ++j) cnt += (fabs(DSUB(pt_dist(P, i, j), LOC_D1)) < LOC_TOL) ? 1 : 0;
        if (cnt < 2) continue;
        bool done = false;
        for (int a = 0; a < K && !done; ++a) {                  // cartesian_product(matches, matches), helpers.py:443
            if (!(fabs(DSUB(pt_dist(P, i, a), LOC_D1)) < LOC_TOL)) continue;
            for (int b = 0; b < K; ++b) {
                if (!(fabs(DSUB(pt_dist(P, i, b), LOC_D1)) < LOC_TOL)) continue;
                if (fabs(DSUB(pt_dist(P, a, b), LOC_D2)) > LOC_TOL) continue;
                // helpers.py:453-455: i, a, b all go on the list that only ever screens i
                if (i < 64) used_lo |= 1ull << i; else used_hi |= 1ull << (i - 64);
                if (a < 64) used_lo |= 1ull << a; else used_hi |= 1ull << (a - 64);
                if (b < 64) used_lo |= 1ull << b; else used_hi |= 1ull << (b - 64);
                const double lx = DADD(P[3 * a], P[3 * b]) / 2.0, ly = DADD(P[3 * a + 1], P[3 * b + 1]) / 2.0, lz = DADD(P[3 * a + 2], P[3 * b + 2]) / 2.0;
                const double e = DADD(DADD(E[i], E[a]), E[b]) / 3.0;
                double hx = DSUB(P[3 * a], P[3 * b]), hy = DSUB(P[3 * a + 1], P[3 * b + 1]), hz = DSUB(P[3 * a + 2], P[3 * b + 2]);
                const double nrm = sqrt(DADD(DADD(DMUL(hx, hx), DMUL(hy, hy)), DMUL(hz, hz)));
                hx /= nrm; hy /= nrm;
                double heading = atan2(hy, hx);
                const double pi = 3.141592653589793;
                if (heading > pi / 2) heading = heading - pi;
                if (heading < -pi / 2) heading = heading + pi;
                if (found < max_objects) {
                    double* o = out + (size_t)found * 5;
                    o[0] = lx; o[1] = ly; o[2] = lz; o[3] = -heading; o[4] = e;
                    drone_index[found] = (DSUB(P[3 * i + 1], ly) > 0.0) ? 0 : 1;
                }
                ++found;
                done = true;
                break;
            }
        }
    }
    return found;
}

// Frame-set s of a batch in the layout of mocap_locate_objects_dev: obj [n_sets][rmax][3], err [n_sets][rmax], n_obj
// [n_sets] (clamped to rmax; <= 0: no points) -> out [n_sets][max_objects][5], drone_index [n_sets][max_objects],
// n_out [n_sets].  Objects found beyond max_objects are dropped in scan order and n_out is clamped to max_objects.
GEOM_HD void locate_frame_set(const double* __restrict__ obj, const double* __restrict__ err, const int32_t* __restrict__ n_obj,
                              int s, int rmax, int max_objects, double* __restrict__ out, int32_t* __restrict__ drone_index,
                              int32_t* __restrict__ n_out) {
    const int K = n_obj[s] < rmax ? n_obj[s] : rmax;
    const int found = locate_scan(obj + (size_t)s * rmax * 3, err + (size_t)s * rmax, K, max_objects,
                                  out + (size_t)s * max_objects * 5, drone_index + (size_t)s * max_objects);
    n_out[s] = found < max_objects ? found : max_objects;
}
