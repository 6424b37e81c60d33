// The detection overlay _find_dot draws into every captured frame (reference computer_code/api/helpers.py:148,156-157),
// as pixel-exact drawing code.  Written against geom.cuh only (no CUDA headers), so that tests/hostcheck/overlay_host.cpp
// runs this very code with g++ and the kernels of overlay.cu run it on the device.
//
// What _find_dot draws reduces to three layers over the frame, in this order:
//   contours  cv.drawContours(img, findContours(RETR_TREE, CHAIN_APPROX_SIMPLE), -1, (0,255,0), 1) paints exactly the
//             foreground pixels (grey > 51) with a 4-neighbour that is background or outside the image (ov_border);
//   marks     per contour with m00 != 0 -- S1's blob list -- in (100,255,100): the label
//             cv.putText(img, '(x, y)', (x, y-15), FONT_HERSHEY_SIMPLEX, 0.3, colour, 1) (ov_label_char) and
//             cv.circle(img, (x, y), 1, colour, -1), a 5-pixel plus (ov_plus).  One colour, so their order is free.
// The grey is the frame's before anything is drawn.
//
// The label follows cv2's putText: FONT_HERSHEY_SIMPLEX strokes (ov_glyph: digits, '(', ')', ',', ' ' and '-'), scaled
// in 16.16 fixed point by cvRound(0.3 * 65536), each stroke a thickness-1 8-connected line between fixed-point end
// points clipped to the image (ov_line_fx).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "geom.cuh"

#define OV_THRESHOLD 51                  // cv.threshold(grey, 255*0.2, 255, THRESH_BINARY) == grey > 51
#define OV_XY_SHIFT 16
#define OV_XY_ONE (1ll << OV_XY_SHIFT)
#define OV_TEXT_SCALE 19661              // cvRound(0.3 * XY_ONE)
#define OV_BASE_LINE (-9)                // FONT_HERSHEY_SIMPLEX's base line, in font units
#define OV_LABEL_DY 15                   // the label's origin is (x, y - 15)
#define OV_MAX_LABEL 26                  // '(' x ', ' y ')' with two 32-bit integers

// contour colour (B, G, R as stored) and the marks' colour
#define OV_CONTOUR_0 0
#define OV_CONTOUR_1 255
#define OV_CONTOUR_2 0
#define OV_MARK_0 100
#define OV_MARK_1 255
#define OV_MARK_2 100

// cvtColor(frame, COLOR_RGB2GRAY) of one 8-bit pixel, byte 0 first: cv2's 15-bit fixed point, as S1 computes it
GEOM_HD int ov_gray(const uint8_t* px) {
    return (px[0] * 9798 + px[1] * 19235 + px[2] * 3735 + 16384) >> 15;
}

// is (x, y) of the W x H grey plane g a contour pixel (foreground with a background or outside 4-neighbour)
GEOM_HD int ov_border(const uint8_t* g, int W, int H, int x, int y) {
    const uint8_t* p = g + (size_t)y * W + x;
    if (p[0] <= OV_THRESHOLD) return 0;
    if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return 1;
    return p[-1] <= OV_THRESHOLD || p[1] <= OV_THRESHOLD || p[-W] <= OV_THRESHOLD || p[W] <= OV_THRESHOLD;
}

GEOM_HD void ov_put(uint8_t* frame, int W, int H, int x, int y, uint8_t c0, uint8_t c1, uint8_t c2) {
    if (x < 0 || y < 0 || x >= W || y >= H) return;
    uint8_t* px = frame + ((size_t)y * W + x) * 3;
    px[0] = c0; px[1] = c1; px[2] = c2;
}

// cv.circle(img, (x, y), 1, colour, -1): the centre and its 4 neighbours inside the frame
GEOM_HD void ov_plus(uint8_t* frame, int W, int H, int x, int y) {
    ov_put(frame, W, H, x, y, OV_MARK_0, OV_MARK_1, OV_MARK_2);
    ov_put(frame, W, H, x - 1, y, OV_MARK_0, OV_MARK_1, OV_MARK_2);
    ov_put(frame, W, H, x + 1, y, OV_MARK_0, OV_MARK_1, OV_MARK_2);
    ov_put(frame, W, H, x, y - 1, OV_MARK_0, OV_MARK_1, OV_MARK_2);
    ov_put(frame, W, H, x, y + 1, OV_MARK_0, OV_MARK_1, OV_MARK_2);
}

// cv2's clipLine on a w x h rectangle (in the segment's units); 0: nothing of the segment is inside
GEOM_HD int ov_clip(int64_t w, int64_t h, int64_t* x1, int64_t* y1, int64_t* x2, int64_t* y2) {
    const int64_t right = w - 1, bottom = h - 1;
    int c1 = (*x1 < 0) + (*x1 > right) * 2 + (*y1 < 0) * 4 + (*y1 > bottom) * 8;
    int c2 = (*x2 < 0) + (*x2 > right) * 2 + (*y2 < 0) * 4 + (*y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        int64_t a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            *x1 += (int64_t)((double)(a - *y1) * (double)(*x2 - *x1) / (double)(*y2 - *y1));
            *y1 = a;
            c1 = (*x1 < 0) + (*x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            *x2 += (int64_t)((double)(a - *y2) * (double)(*x2 - *x1) / (double)(*y2 - *y1));
            *y2 = a;
            c2 = (*x2 < 0) + (*x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                *y1 += (int64_t)((double)(a - *x1) * (double)(*y2 - *y1) / (double)(*x2 - *x1));
                *x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                *y2 += (int64_t)((double)(a - *x2) * (double)(*y2 - *y1) / (double)(*x2 - *x1));
                *x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// cv::line(img, p1, p2, colour, 1, LINE_8) between integer end points: clipped to the frame by cv2's clipLine, then
// Bresenham's 8-connected walk from the left end point (cv2's LineIterator); lane `lane` of `lanes` paints every
// lanes-th pixel of the walk
GEOM_HD void ov_line(uint8_t* frame, int W, int H, int64_t x1, int64_t y1, int64_t x2, int64_t y2, uint8_t c0, uint8_t c1, uint8_t c2,
                     int lane = 0, int lanes = 1) {
    if (!ov_clip(W, H, &x1, &y1, &x2, &y2)) return;
    int x = (int)x1, y = (int)y1;
    int dx = (int)(x2 - x1), dy = (int)(y2 - y1);
    if (dx < 0) { dx = -dx; dy = -dy; x = (int)x2; y = (int)y2; }
    const int sy = dy < 0 ? -1 : 1;
    if (dy < 0) dy = -dy;
    const int steep = dy > dx;
    if (steep) { const int t = dx; dx = dy; dy = t; }
    // the major axis steps every pixel, the minor one when err goes negative
    int err = dx - (dy + dy);
    const int plus = dx + dx, minus = -(dy + dy);
    for (int k = 0; k <= dx; ++k) {
        if (k % lanes == lane) ov_put(frame, W, H, x, y, c0, c1, c2);
        const int mask = err < 0;
        err += minus + (mask ? plus : 0);
        if (steep) { y += sy; x += mask; } else { x += 1; y += mask ? sy : 0; }
    }
}

// a putText stroke between 16.16 fixed-point end points: rounded to whole pixels, then ov_line
GEOM_HD void ov_line_fx(uint8_t* frame, int W, int H, int64_t x1, int64_t y1, int64_t x2, int64_t y2) {
    const int64_t h = OV_XY_ONE >> 1;
    ov_line(frame, W, H, (x1 + h) >> OV_XY_SHIFT, (y1 + h) >> OV_XY_SHIFT, (x2 + h) >> OV_XY_SHIFT, (y2 + h) >> OV_XY_SHIFT,
            OV_MARK_0, OV_MARK_1, OV_MARK_2);
}

// the strokes of one Hershey glyph in cv2's encoding: two characters of left and right bearing, then vertices as
// character pairs (coordinate + 'R'), a space lifting the pen; drawn with its left bearing at the 16.16 pen position
// *view_x, which moves on by the glyph's advance
GEOM_HD void ov_glyph_draw(uint8_t* frame, int W, int H, const char* g, int64_t* view_x, int64_t view_y, int64_t scale) {
    const int64_t left = g[0] - 'R', right = g[1] - 'R';
    *view_x -= left * scale;
    int64_t px = 0, py = 0;
    int have = 0;
    for (const char* p = g + 2;; ) {
        if (*p == ' ' || !*p) {
            have = 0;
            if (!*p++) break;
        } else {
            const int64_t x = (p[0] - 'R') * scale + *view_x, y = (p[1] - 'R') * scale + view_y;
            p += 2;
            if (have) ov_line_fx(frame, W, H, px, py, x, y);
            px = x; py = y; have = 1;
        }
    }
    *view_x += right * scale;
}

// FONT_HERSHEY_SIMPLEX glyphs of the characters a label holds, as cv2 renders them (pinned against cv2.putText by
// tests/test_overlay_on_host.py); NULL for any other character
GEOM_HD const char* ov_glyph(char c) {
    switch (c) {
        case ' ': return "JZ";
        case '(': return "KYVBTDRGPKOPOTPYR]T`Vb";
        case ')': return "KYNBPDRGTKUPUTTYR]P`Nb";
        case ',': return "MWSZR[QZRYSZS\\R^Q_";
        case '-': return "E_IR[R";
        case '0': return "H\\QFNGLJKOKRLWNZQ[S[VZXWYRYOXJVGSFQF";
        case '1': return "H\\NJPISFS[";
        case '2': return "H\\LKLJMHNGPFTFVGWHXJXLWNUQK[Y[";
        case '3': return "H\\MFXFRNUNWOXPYSYUXXVZS[P[MZLYKW";
        case '4': return "H\\UFKTZT UFU[";
        case '5': return "H\\WFMFLOMNPMSMVNXPYSYUXXVZS[P[MZLYKW";
        case '6': return "H\\XIWGTFRFOGMJLOLTMXOZR[S[VZXXYUYTXQVOSNRNOOMQLT";
        case '7': return "H\\YFO[ KFYF";
        case '8': return "H\\PFMGLILKMMONSOVPXRYTYWXYWZT[P[MZLYKWKTLRNPQOUNWMXKXIWGTFPF";
        case '9': return "H\\XMWPURRSQSNRLPKMKLLINGQFRFUGWIXMXRWWUZR[P[MZLX";
        default: return nullptr;
    }
}

// the label '(x, y)' of a blob centre: its characters into s (at least OV_MAX_LABEL), returns their count
GEOM_HD int ov_label_text(int x, int y, char* s) {
    int n = 0;
    s[n++] = '(';
    for (int k = 0; k < 2; ++k) {
        const int v = k ? y : x;
        unsigned int u = v < 0 ? 0u - (unsigned int)v : (unsigned int)v;
        char d[10];
        int nd = 0;
        do { d[nd++] = (char)('0' + u % 10); u /= 10; } while (u);
        if (v < 0) s[n++] = '-';
        while (nd) s[n++] = d[--nd];
        if (!k) { s[n++] = ','; s[n++] = ' '; }
    }
    s[n++] = ')';
    return n;
}

// character k of the label of the blob centred at (x, y): cv.putText(img, f'({x}, {y})', (x, y - 15),
// FONT_HERSHEY_SIMPLEX, 0.3, (100, 255, 100), 1).  Returns 0 when the label has no character k.
GEOM_HD int ov_label_char(uint8_t* frame, int W, int H, int x, int y, int k) {
    char s[OV_MAX_LABEL];
    const int n = ov_label_text(x, y, s);
    if (k >= n) return 0;
    int64_t view_x = (int64_t)x * OV_XY_ONE;
    const int64_t view_y = (int64_t)(y - OV_LABEL_DY) * OV_XY_ONE + (int64_t)OV_BASE_LINE * OV_TEXT_SCALE;
    for (int i = 0; i < k; ++i) {
        const char* g = ov_glyph(s[i]);
        view_x += (int64_t)(g[1] - g[0]) * OV_TEXT_SCALE;
    }
    ov_glyph_draw(frame, W, H, ov_glyph(s[k]), &view_x, view_y, OV_TEXT_SCALE);
    return 1;
}

// the whole marks layer of one blob: its label and its plus
GEOM_HD void ov_marks(uint8_t* frame, int W, int H, int x, int y) {
    for (int k = 0; ov_label_char(frame, W, H, x, y, k); ++k) {}
    ov_plus(frame, W, H, x, y);
}

// drawlines' end points of the float32 line (a, b, c) in a frame `width` pixels wide (helpers.py:497-503):
// (0, int(-c / b)) and (width, int(-(c + a * width) / b)), float32 arithmetic, int() truncating.  Returns 0 where the
// reference raises instead of drawing: b == 0 or another non-finite end point (int() of inf or NaN), or an end point
// outside cv.line's 32-bit range.
GEOM_HD int ov_epiline_ends(float a, float b, float c, int width, int64_t* y0, int64_t* y1) {
#ifdef __CUDA_ARCH__
    const float f0 = __fdiv_rn(-c, b), f1 = __fdiv_rn(-__fadd_rn(c, __fmul_rn(a, (float)width)), b);
#else
    const float f0 = -c / b, f1 = -(c + a * (float)width) / b;
#endif
    // as floats: a finite float below 2^31 in magnitude truncates into the range; -2^31 itself is in it
    if (!(f0 > -2147483904.0f && f0 < 2147483648.0f) || !(f1 > -2147483904.0f && f1 < 2147483648.0f)) return 0;
    *y0 = (int64_t)f0;
    *y1 = (int64_t)f1;
    return 1;
}

// the palette of the epipolar lines: numpy's np.random.RandomState(seed).randint(0, 255, (n, 3)) -- MT19937 seeded
// by init_genrand, each value the low 8 bits of one 32-bit draw, drawn again while above 254 -- so that line k of a
// session has the colour the reference's k-th np.random.randint(0, 255, 3) gives after np.random.seed(seed)
static inline void ov_palette(uint32_t seed, int n, uint8_t* out) {
    uint32_t mt[624];
    mt[0] = seed;
    for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    int idx = 624;
    for (int k = 0; k < 3 * n; ++k) {
        uint32_t v;
        do {
            if (idx == 624) {
                for (int i = 0; i < 624; ++i) {
                    const uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
                    mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
                }
                idx = 0;
            }
            uint32_t y = mt[idx++];
            y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
            v = y & 255u;
        } while (v > 254u);
        out[k] = (uint8_t)v;
    }
}

