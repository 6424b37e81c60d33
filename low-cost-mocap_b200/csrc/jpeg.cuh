// Baseline JPEG encoding as cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) drives libjpeg-turbo: BGR uint8 in,
// 4:2:0 (MCU of 16 x 16 pixels: Y00 Y01 Y10 Y11 Cb Cr), the Annex K Huffman tables, no restart markers.  Written
// against geom.cuh only (no CUDA headers), so that tests/hostcheck/jpeg_host.cpp runs this very code with g++ and the
// kernels of jpeg.cu run it per block / per MCU.
//
// The libjpeg conventions reproduced (DESIGN.md section 10):
//   colour   jccolor.c: 16-bit fixed point, ONE_HALF on Y, CBCR_OFFSET + ONE_HALF - 1 on Cb / Cr;
//   edges    the right edge replicated to ceil(w/8)*8 (Y) and to ceil(w/16)*16 before downsampling (Cb / Cr), the last
//            row replicated to an even row count before downsampling, then the last downsampled row (jcprepct.c);
//   chroma   h2v2_downsample: (sum of 2 x 2 + bias) >> 2, bias 1, 2, 1, 2, ... along the output row;
//   DCT      jfdctint.c (6b islow): CONST_BITS 13, PASS1_BITS 2, output scaled by 8;
//   quantise compute_reciprocal (jcdctmgr.c, 16-bit DCTELEM): ((|x| + corr) * recip) >> shift for divisor 8 * table;
//   dummies  luma blocks of the last MCU column / row past ceil(w/8) / ceil(h/8): AC 0, DC of the block before them
//            in the MCU (jccoefct.c compress_data);
//   entropy  jchuff.c: ZRL only before a non-zero coefficient, no EOB after a non-zero coefficient 63, the tail padded
//            with 1-bits, 0x00 stuffed after every 0xFF.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "geom.cuh"

#define JPEG_HEADER_BYTES  623         // SOI 2, APP0 18, DQT 2 x 69, SOF0 19, DHT 2 x 33 + 2 x 183, SOS 14
#define JPEG_EOI_BYTES     2
#define JPEG_BLOCK_MAX_BITS 1660       // DC 11 + 11 (chroma code of category 11), then 63 x (16 + 10)
#define JPEG_MCU_MAX_BITS  (6 * JPEG_BLOCK_MAX_BITS)
#define JPEG_MAX_DIM       65500       // JPEG_MAX_DIMENSION of libjpeg

// Tables of one quality, built on the host (jpeg_build_tables) and copied to the device with the header.
struct JpegTables {
    uint16_t recip[2][64];             // natural order; [0] luma, [1] chroma
    uint16_t corr[2][64];
    uint8_t  shift[2][64];
    uint8_t  natural[64];              // natural index of zigzag position k
    uint16_t dc_code[2][12];
    uint8_t  dc_len[2][12];
    uint16_t ac_code[2][256];
    uint8_t  ac_len[2][256];
};

// ---------------------------------------------------------------------------------------------- pixels
GEOM_HD void jpeg_ycc(int b, int g, int r, int* y, int* cb, int* cr) {
    // FIX(x) = (int)(x * 65536 + 0.5)
    *y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    *cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    *cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// Pixel (y, x) of an image viewed as `tiles` frames of tile_h x tile_w x 3 side by side (np.hstack of the frames, the
// frames stored one after another): W = tiles * tile_w, H = tile_h.
GEOM_HD const uint8_t* jpeg_pixel(const uint8_t* img, int tile_w, int tile_h, int y, int x) {
    const int t = x / tile_w;
    return img + (((size_t)t * tile_h + y) * tile_w + (x - t * tile_w)) * 3;
}

// The 64 samples block `blk` (0-3 luma, 4 Cb, 5 Cr) of MCU (mx, my) reads, padded as libjpeg pads.
GEOM_HD void jpeg_block_samples(const uint8_t* img, int tile_w, int tile_h, int W, int mx, int my, int blk, int* s) {
    const int H = tile_h;
    if (blk < 4) {
        const int y0 = my * 16 + (blk >> 1) * 8, x0 = mx * 16 + (blk & 1) * 8;
        for (int i = 0; i < 8; ++i) {
            const int y = y0 + i < H ? y0 + i : H - 1;
            for (int j = 0; j < 8; ++j) {
                const int x = x0 + j < W ? x0 + j : W - 1;
                const uint8_t* p = jpeg_pixel(img, tile_w, tile_h, y, x);
                int Y, cb, cr;
                jpeg_ycc(p[0], p[1], p[2], &Y, &cb, &cr);
                s[i * 8 + j] = Y;
            }
        }
        return;
    }
    const int last_row = (H + 1) / 2 - 1;             // the last downsampled row; rows past it repeat it
    for (int i = 0; i < 8; ++i) {
        int cy = my * 8 + i;
        if (cy > last_row) cy = last_row;
        for (int j = 0; j < 8; ++j) {
            const int cx = mx * 8 + j;
            int sum = 0;
            for (int dy = 0; dy < 2; ++dy)
                for (int dx = 0; dx < 2; ++dx) {
                    const int y = 2 * cy + dy < H ? 2 * cy + dy : H - 1;
                    const int x = 2 * cx + dx < W ? 2 * cx + dx : W - 1;
                    const uint8_t* p = jpeg_pixel(img, tile_w, tile_h, y, x);
                    int Y, cb, cr;
                    jpeg_ycc(p[0], p[1], p[2], &Y, &cb, &cr);
                    sum += blk == 4 ? cb : cr;
                }
            s[i * 8 + j] = (sum + 1 + (cx & 1)) >> 2;
        }
    }
}

// ---------------------------------------------------------------------------------------------- DCT, quantisation
#define JPEG_DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))

// One 8-point pass of jfdctint.c over d[0], d[step], ..., d[7 * step].  Every intermediate fits 32 bits: the column
// pass's largest product is (z3 + z4) * FIX_1_175875602 with |z3 + z4| <= 32768.
GEOM_HD void jpeg_fdct_pass(int* d, int step, int first) {
    const int t0 = d[0] + d[7 * step], t7 = d[0] - d[7 * step];
    const int t1 = d[step] + d[6 * step], t6 = d[step] - d[6 * step];
    const int t2 = d[2 * step] + d[5 * step], t5 = d[2 * step] - d[5 * step];
    const int t3 = d[3 * step] + d[4 * step], t4 = d[3 * step] - d[4 * step];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    const int n = first ? 13 - 2 : 13 + 2;
    if (first) {
        d[0] = (t10 + t11) * 4;
        d[4 * step] = (t10 - t11) * 4;
    } else {
        d[0] = JPEG_DESCALE(t10 + t11, 2);
        d[4 * step] = JPEG_DESCALE(t10 - t11, 2);
    }
    int z1 = (t12 + t13) * 4433;
    d[2 * step] = JPEG_DESCALE(z1 + t13 * 6270, n);
    d[6 * step] = JPEG_DESCALE(z1 - t12 * 15137, n);
    z1 = t4 + t7;
    int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
    const int z5 = (z3 + z4) * 9633;
    const int a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
    z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
    d[7 * step] = JPEG_DESCALE(a4 + z1 + z3, n);
    d[5 * step] = JPEG_DESCALE(a5 + z2 + z4, n);
    d[3 * step] = JPEG_DESCALE(a6 + z2 + z3, n);
    d[step] = JPEG_DESCALE(a7 + z1 + z4, n);
}

// samples s[64] (0..255, natural order) -> jpeg_fdct_islow output in place
GEOM_HD void jpeg_fdct(int* s) {
    for (int i = 0; i < 64; ++i) s[i] -= 128;
    for (int r = 0; r < 8; ++r) jpeg_fdct_pass(s + r * 8, 1, 1);
    for (int c = 0; c < 8; ++c) jpeg_fdct_pass(s + c, 8, 0);
}

// fdct output d[64] (natural) -> quantised coefficients in zigzag order
GEOM_HD void jpeg_quantize(const int* d, const JpegTables& T, int t, int16_t* zz) {
    for (int k = 0; k < 64; ++k) {
        const int i = T.natural[k];
        const int x = d[i];
        const uint32_t a = (uint32_t)(x < 0 ? -x : x);
        const int q = (int)(((a + T.corr[t][i]) * (uint32_t)T.recip[t][i]) >> T.shift[t][i]);
        zz[k] = (int16_t)(x < 0 ? -q : q);
    }
}

// ---------------------------------------------------------------------------------------------- entropy coding
GEOM_HD int jpeg_nbits(int v) {
    int a = v < 0 ? -v : v, n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}

GEOM_HD int jpeg_dc_bits(int diff, const JpegTables& T, int t) {
    const int s = jpeg_nbits(diff);
    return T.dc_len[t][s] + s;
}

// bits of a block's AC codes: ZRLs, (run, size) codes with their extra bits, EOB
GEOM_HD int jpeg_ac_bits(const int16_t* zz, const JpegTables& T, int t) {
    int bits = 0, run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = zz[k];
        if (!v) { ++run; continue; }
        for (; run > 15; run -= 16) bits += T.ac_len[t][0xF0];
        const int s = jpeg_nbits(v);
        bits += T.ac_len[t][(run << 4) | s] + s;
        run = 0;
    }
    if (run) bits += T.ac_len[t][0];
    return bits;
}

// Table of each block of the MCU, and whether it is a dummy (mw, mh: MCUs across / down; wb, hb: luma blocks).
GEOM_HD int jpeg_table_of(int blk) { return blk < 4 ? 0 : 1; }

GEOM_HD int jpeg_is_dummy(int blk, int mx, int my, int wb, int hb) {
    if (blk >= 4) return 0;
    return (2 * mx + (blk & 1) >= wb) || (2 * my + (blk >> 1) >= hb);
}

// The quantised DCs of an MCU's blocks as libjpeg codes them: a dummy takes the DC of the block before it in the MCU.
// raw[6]: what the DCT gave (ignored for dummies).
GEOM_HD void jpeg_mcu_dc(const int* raw, int mx, int my, int wb, int hb, int* dc) {
    for (int b = 0; b < 6; ++b) dc[b] = (b > 0 && jpeg_is_dummy(b, mx, my, wb, hb)) ? dc[b - 1] : raw[b];
}

// DC differences of MCU m's blocks in scan order, from an image's coefficients [n_mcu][6][64] (zigzag): the luma
// predictor runs through Y00 Y01 Y10 Y11 of each MCU in turn, Cb and Cr have their own, all starting at 0.
GEOM_HD void jpeg_mcu_diffs(const int16_t* coef, int m, int mw, int wb, int hb, int* diff) {
    int raw[6], cur[6], prv[6] = {0, 0, 0, 0, 0, 0};
    for (int b = 0; b < 6; ++b) raw[b] = coef[((size_t)m * 6 + b) * 64];
    jpeg_mcu_dc(raw, m % mw, m / mw, wb, hb, cur);
    if (m > 0) {
        for (int b = 0; b < 6; ++b) raw[b] = coef[((size_t)(m - 1) * 6 + b) * 64];
        jpeg_mcu_dc(raw, (m - 1) % mw, (m - 1) / mw, wb, hb, prv);
    }
    diff[0] = cur[0] - prv[3];
    diff[1] = cur[1] - cur[0];
    diff[2] = cur[2] - cur[1];
    diff[3] = cur[3] - cur[2];
    diff[4] = cur[4] - prv[4];
    diff[5] = cur[5] - prv[5];
}

// Bit writer of one MCU's codes into a word array (MSB first within big-endian 32-bit words) from bit `off`.  Words
// the MCU shares with its neighbours (the first when `off` is not word aligned, the last when its end is not) are
// OR-ed in, atomically on the device; words it owns whole are plain stores.  The word array is zero where OR-ed.
struct JpegBitWriter {
    uint32_t* words;
    uint64_t word;                     // index of the word acc's top 32 bits go to
    uint64_t acc;                      // pending bits, MSB first from bit 63
    int n;                             // pending bits in acc, the shared leading bits of the first word included
    int shared;                        // the next word emitted is shared
};

GEOM_HD void jpeg_store(uint32_t* w, uint32_t v, int shared) {
#if defined(__CUDA_ARCH__)
    if (shared) atomicOr(w, v); else *w = v;
#else
    if (shared) *w |= v; else *w = v;
#endif
}

GEOM_HD void jpeg_bw_init(JpegBitWriter* bw, uint32_t* words, uint64_t off) {
    bw->words = words;
    bw->word = off >> 5;
    bw->acc = 0;
    bw->n = (int)(off & 31);
    bw->shared = bw->n != 0;
}

GEOM_HD void jpeg_bw_put(JpegBitWriter* bw, uint32_t v, int len) {   // len <= 27
    if (!len) return;
    bw->acc |= (uint64_t)v << (64 - bw->n - len);
    bw->n += len;
    if (bw->n >= 32) {
        jpeg_store(bw->words + bw->word, (uint32_t)(bw->acc >> 32), bw->shared);
        bw->acc <<= 32;
        bw->n -= 32;
        bw->word += 1;
        bw->shared = 0;
    }
}

GEOM_HD void jpeg_bw_flush(JpegBitWriter* bw) {
    if (bw->n) jpeg_store(bw->words + bw->word, (uint32_t)(bw->acc >> 32), 1);
}

GEOM_HD uint32_t jpeg_extra(int v, int s) {
    return (uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1);
}

GEOM_HD void jpeg_put_block(JpegBitWriter* bw, const int16_t* zz, int diff, const JpegTables& T, int t) {
    int s = jpeg_nbits(diff);
    jpeg_bw_put(bw, ((uint32_t)T.dc_code[t][s] << s) | jpeg_extra(diff, s), T.dc_len[t][s] + s);
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = zz[k];
        if (!v) { ++run; continue; }
        for (; run > 15; run -= 16) jpeg_bw_put(bw, T.ac_code[t][0xF0], T.ac_len[t][0xF0]);
        s = jpeg_nbits(v);
        const int sym = (run << 4) | s;
        jpeg_bw_put(bw, ((uint32_t)T.ac_code[t][sym] << s) | jpeg_extra(v, s), T.ac_len[t][sym] + s);
        run = 0;
    }
    if (run) jpeg_bw_put(bw, T.ac_code[t][0], T.ac_len[t][0]);
}

// byte j of the big-endian word array
GEOM_HD uint8_t jpeg_byte(const uint32_t* words, uint64_t j) {
    return (uint8_t)(words[j >> 2] >> (24 - 8 * (int)(j & 3)));
}

// 0xFF bytes among entropy bytes [j0, j1)
GEOM_HD uint64_t jpeg_count_ff(const uint32_t* words, uint64_t j0, uint64_t j1) {
    uint64_t n = 0;
    for (uint64_t j = j0; j < j1; ++j) n += jpeg_byte(words, j) == 0xFF;
    return n;
}

// entropy bytes [j0, j1) to out[at...], a 0x00 after each 0xFF; at = j0 + the 0xFF bytes before j0
GEOM_HD void jpeg_stuff(const uint32_t* words, uint64_t j0, uint64_t j1, uint8_t* out, uint64_t at) {
    for (uint64_t j = j0; j < j1; ++j) {
        const uint8_t v = jpeg_byte(words, j);
        out[at++] = v;
        if (v == 0xFF) out[at++] = 0;
    }
}

// ---------------------------------------------------------------------------------------------- host side
static const uint8_t JPEG_QUANT_BASE[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
     47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
static const uint8_t JPEG_DC_BITS[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                            {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t JPEG_AC_BITS[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                            {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t JPEG_AC_VALS[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
     0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
     0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
     0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
     0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
     0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
     0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
     0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
     0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
     0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
     0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
     0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
     0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
     0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
     0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
     0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
     0xf9, 0xfa}};

// jpeg_set_quality(cinfo, quality, force_baseline = TRUE) -> quant[2][64] in natural order
static inline void jpeg_quant_tables(int quality, uint8_t quant[2][64]) {
    const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int t = 0; t < 2; ++t)
        for (int i = 0; i < 64; ++i) {
            long v = ((long)JPEG_QUANT_BASE[t][i] * scale + 50) / 100;
            quant[t][i] = (uint8_t)(v < 1 ? 1 : v > 255 ? 255 : v);
        }
}

static inline void jpeg_zigzag(uint8_t natural[64]) {
    int k = 0;
    for (int s = 0; s < 15; ++s) {
        const int lo = s < 8 ? 0 : s - 7, hi = s < 8 ? s : 7;      // rows on anti-diagonal s
        for (int j = 0; j <= hi - lo; ++j) {
            const int r = (s & 1) ? lo + j : hi - j;                   // even diagonals run upwards
            natural[k++] = (uint8_t)(r * 8 + (s - r));
        }
    }
}

static inline void jpeg_huff_codes(const uint8_t* bits, const uint8_t* vals, uint16_t* code, uint8_t* len) {
    int c = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < bits[l - 1]; ++i, ++k) {
            code[vals[k]] = (uint16_t)c++;
            len[vals[k]] = (uint8_t)l;
        }
        c <<= 1;
    }
}

static inline void jpeg_build_tables(int quality, JpegTables* T) {
    uint8_t quant[2][64];
    jpeg_quant_tables(quality, quant);
    jpeg_zigzag(T->natural);
    for (int t = 0; t < 2; ++t) {
        for (int i = 0; i < 64; ++i) {                                // compute_reciprocal, divisor 8 * table >= 8
            const uint32_t d = 8u * quant[t][i];
            int b = 0;
            while ((d >> (b + 1)) != 0) ++b;
            int r = 16 + b;
            uint64_t fq = ((uint64_t)1 << r) / d, fr = ((uint64_t)1 << r) % d;
            uint32_t c = d / 2;
            if (fr == 0) { fq >>= 1; --r; }
            else if (fr <= d / 2) ++c;
            else ++fq;
            T->recip[t][i] = (uint16_t)fq;
            T->corr[t][i] = (uint16_t)c;
            T->shift[t][i] = (uint8_t)r;
        }
        uint8_t dc_vals[12];
        for (int i = 0; i < 12; ++i) dc_vals[i] = (uint8_t)i;
        memset(T->dc_len[t], 0, sizeof T->dc_len[t]);
        memset(T->ac_len[t], 0, sizeof T->ac_len[t]);
        jpeg_huff_codes(JPEG_DC_BITS[t], dc_vals, T->dc_code[t], T->dc_len[t]);
        jpeg_huff_codes(JPEG_AC_BITS[t], JPEG_AC_VALS[t], T->ac_code[t], T->ac_len[t]);
    }
}

static inline uint8_t* jpeg_put16(uint8_t* p, int v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; return p + 2; }

// SOI .. SOS of one image, JPEG_HEADER_BYTES bytes, in libjpeg's order
static inline void jpeg_build_header(int width, int height, int quality, uint8_t* h) {
    static const uint8_t app0[20] = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    uint8_t quant[2][64], natural[64];
    jpeg_quant_tables(quality, quant);
    jpeg_zigzag(natural);
    uint8_t* p = h;
    memcpy(p, app0, sizeof app0); p += sizeof app0;
    for (int t = 0; t < 2; ++t) {
        *p++ = 0xFF; *p++ = 0xDB; p = jpeg_put16(p, 67); *p++ = (uint8_t)t;
        for (int k = 0; k < 64; ++k) *p++ = quant[t][natural[k]];
    }
    *p++ = 0xFF; *p++ = 0xC0; p = jpeg_put16(p, 17); *p++ = 8;
    p = jpeg_put16(p, height); p = jpeg_put16(p, width);
    static const uint8_t comps[10] = {3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
    memcpy(p, comps, sizeof comps); p += sizeof comps;
    for (int t = 0; t < 2; ++t) {
        *p++ = 0xFF; *p++ = 0xC4; p = jpeg_put16(p, 3 + 16 + 12); *p++ = (uint8_t)t;
        memcpy(p, JPEG_DC_BITS[t], 16); p += 16;
        for (int i = 0; i < 12; ++i) *p++ = (uint8_t)i;
        *p++ = 0xFF; *p++ = 0xC4; p = jpeg_put16(p, 3 + 16 + 162); *p++ = (uint8_t)(0x10 | t);
        memcpy(p, JPEG_AC_BITS[t], 16); p += 16;
        memcpy(p, JPEG_AC_VALS[t], 162); p += 162;
    }
    static const uint8_t sos[14] = {0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 0x3F, 0};
    memcpy(p, sos, sizeof sos);
}

// worst-case bytes of one image: the header, every MCU at its largest, each byte stuffed, EOI
static inline uint64_t jpeg_bound(int width, int height) {
    const uint64_t mcus = (uint64_t)((width + 15) / 16) * (uint64_t)((height + 15) / 16);
    return JPEG_HEADER_BYTES + 2 * ((mcus * JPEG_MCU_MAX_BITS + 7) / 8) + JPEG_EOI_BYTES;
}
