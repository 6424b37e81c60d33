// One read of the live capture loop, per frame-set: the part of Cameras._camera_read (reference
// computer_code/api/helpers.py:84-92) that sits between S1 and the matcher.  Written against geom.cuh only (no CUDA
// headers), so that tests/hostcheck/live_host.cpp runs this very code with g++ and k_live_blobs (live.cu) runs it with
// one thread per read.
//
// Per camera: the blob count S1 left and its first blob's centre, (-1, -1) when there is none -- the capture-mode
// payload [x[0] for x in image_points] (helpers.py:92), S1's blobs being in cv.findContours order.
// Per read:
//   gate   = some camera has at least one blob: any(np.all(point[0] != [None, None]) ...) (helpers.py:90), the
//            condition under which the reference matches, emits and calls predict_location;
//   called = gate in locate mode, else 0: the reads that are a predict_location call (helpers.py:106);
//   flags  = the OR of the images' MOCAP_F_* bits, and of what the matcher already left in the slot (merge != 0).
// Dots: _find_dot's cv.circle(img, centre, 1, (100, 255, 100), -1) reduced to the 1-px dot the drop-in find_dot draws
// (api.find_dot), at every blob centre inside the S x S frame.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "geom.cuh"

// mode bits (include/mocap_b200.h)
#define LIVE_CAPTURE     1
#define LIVE_TRIANGULATE 2
#define LIVE_LOCATE      4

// blob_xy [C][MB][2], blob_n [C], img_flags [C] of one read (have_blobs == 0: S1 did not run, no blob anywhere).
// Out: cnt [C], first [C][2], *gate, *called, *flags.
GEOM_HD void live_read(int C, int MB, const int32_t* blob_xy, const int32_t* blob_n, const int32_t* img_flags, int have_blobs,
                       int locate, int merge, int32_t* cnt, int32_t* first, uint8_t* gate, uint8_t* called, int32_t* flags) {
    int open = 0, f = merge ? *flags : 0;
    for (int c = 0; c < C; ++c) {
        const int n = have_blobs ? blob_n[c] : 0;
        cnt[c] = n;
        first[2 * c] = n > 0 ? blob_xy[(size_t)c * MB * 2] : -1;
        first[2 * c + 1] = n > 0 ? blob_xy[(size_t)c * MB * 2 + 1] : -1;
        open |= n > 0;
        if (have_blobs) f |= img_flags[c];
    }
    *gate = (uint8_t)open;
    *called = (uint8_t)(locate && open);
    *flags = f;
}

// the dots of one camera's blobs in its processed frame uint8 [S][S][3]
GEOM_HD void live_dots(int MB, const int32_t* blob_xy, int n, int S, uint8_t* frame) {
    if (n > MB) n = MB;
    for (int b = 0; b < n; ++b) {
        const int x = blob_xy[2 * b], y = blob_xy[2 * b + 1];
        if (x < 0 || y < 0 || x >= S || y >= S) continue;
        uint8_t* px = frame + ((size_t)y * S + x) * 3;
        px[0] = 100; px[1] = 255; px[2] = 100;
    }
}
