// Test-only host build of csrc/jpeg.cuh (the JPEG encoder's step code), so that the device kernels' arithmetic can be
// checked stage by stage on a machine without a GPU.  hc_encode walks an image the way the four kernels of jpeg.cu do,
// one block / MCU / chunk after another.  NOT part of libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include <stdlib.h>
#include <vector>
#include "../../low-cost-mocap_b200/csrc/jpeg.cuh"

extern "C" {
int hc_tables_size() { return (int)sizeof(JpegTables); }
void hc_tables(int quality, JpegTables* T) { jpeg_build_tables(quality, T); }
void hc_header(int w, int h, int quality, uint8_t* out) { jpeg_build_header(w, h, quality, out); }
uint64_t hc_bound(int w, int h) { return jpeg_bound(w, h); }

// px uint8 [n][3] (B, G, R) -> out int32 [n][3] (Y, Cb, Cr)
void hc_ycc(int n, const uint8_t* px, int32_t* out) {
    for (int i = 0; i < n; ++i) jpeg_ycc(px[3 * i], px[3 * i + 1], px[3 * i + 2], &out[3 * i], &out[3 * i + 1], &out[3 * i + 2]);
}

// the samples every block of every MCU reads: out int32 [n_mcu][6][64] (dummies included)
void hc_samples(const uint8_t* img, int tiles, int tile_w, int tile_h, int32_t* out) {
    const int W = tiles * tile_w, mw = (W + 15) / 16, mh = (tile_h + 15) / 16;
    for (int m = 0; m < mw * mh; ++m)
        for (int b = 0; b < 6; ++b) jpeg_block_samples(img, tile_w, tile_h, W, m % mw, m / mw, b, out + ((size_t)m * 6 + b) * 64);
}

void hc_fdct(int n, const int32_t* in, int32_t* out) {
    for (int i = 0; i < n; ++i) {
        int d[64];
        for (int k = 0; k < 64; ++k) d[k] = in[(size_t)i * 64 + k];
        jpeg_fdct(d);
        for (int k = 0; k < 64; ++k) out[(size_t)i * 64 + k] = d[k];
    }
}

void hc_quantize(int n, int quality, const int32_t* tabs, const int32_t* d, int16_t* zz) {
    JpegTables T;
    jpeg_build_tables(quality, &T);
    for (int i = 0; i < n; ++i) jpeg_quantize(d + (size_t)i * 64, T, tabs[i], zz + (size_t)i * 64);
}

// per block: DC bits of diffs[i] and AC bits of zz[i], table tabs[i]
void hc_block_bits(int n, const int16_t* zz, const int32_t* diffs, const int32_t* tabs, int32_t* dc, int32_t* ac) {
    JpegTables T;
    jpeg_build_tables(95, &T);
    for (int i = 0; i < n; ++i) {
        dc[i] = jpeg_dc_bits(diffs[i], T, tabs[i]);
        ac[i] = jpeg_ac_bits(zz + (size_t)i * 64, T, tabs[i]);
    }
}

// every block with a bit writer of its own from offs[i] (the words the blocks share are OR-ed), the tail padded with
// 1-bits as k_jpeg_scan pads it; words must hold the stream and be zero
void hc_pack(int n, const int16_t* zz, const int32_t* diffs, const int32_t* tabs, const uint64_t* offs, uint64_t total, uint32_t* words) {
    JpegTables T;
    jpeg_build_tables(95, &T);
    if (total & 7) {
        const int nb = 8 - (int)(total & 7), at = (int)(total & 31);
        words[total >> 5] |= ((1u << nb) - 1) << (32 - at - nb);
    }
    for (int i = 0; i < n; ++i) {
        JpegBitWriter bw;
        jpeg_bw_init(&bw, words, offs[i]);
        jpeg_put_block(&bw, zz + (size_t)i * 64, diffs[i], T, tabs[i]);
        jpeg_bw_flush(&bw);
    }
}

// entropy bytes [0, nbytes) of words -> out with 0x00 after each 0xFF, in chunks placed by an exclusive scan of their
// 0xFF counts as k_jpeg_emit places them; returns the stuffed length
uint64_t hc_stuff(const uint32_t* words, uint64_t nbytes, int chunk, uint8_t* out) {
    uint64_t carry = 0;
    for (uint64_t j0 = 0; j0 < nbytes; j0 += (uint64_t)chunk) {
        const uint64_t j1 = j0 + chunk < nbytes ? j0 + chunk : nbytes;
        jpeg_stuff(words, j0, j1, out, carry + j0);
        carry += jpeg_count_ff(words, j0, j1);
    }
    return nbytes + carry;
}

// the whole encoder, stage by stage as the kernels run it; returns the length, or -1 when it exceeds cap
int64_t hc_encode(const uint8_t* img, int tiles, int tile_w, int tile_h, int quality, uint8_t* out, uint64_t cap) {
    JpegTables T;
    jpeg_build_tables(quality, &T);
    const int W = tiles * tile_w, mw = (W + 15) / 16, mh = (tile_h + 15) / 16, wb = (W + 7) / 8, hb = (tile_h + 7) / 8;
    const int n_mcu = mw * mh;
    std::vector<int16_t> coef((size_t)n_mcu * 6 * 64, 0);
    std::vector<uint16_t> ac((size_t)n_mcu * 6);
    for (int m = 0; m < n_mcu; ++m)                                      // k_jpeg_blocks
        for (int b = 0; b < 6; ++b) {
            int16_t* zz = &coef[((size_t)m * 6 + b) * 64];
            if (jpeg_is_dummy(b, m % mw, m / mw, wb, hb)) { ac[(size_t)m * 6 + b] = T.ac_len[0][0]; continue; }
            int d[64];
            jpeg_block_samples(img, tile_w, tile_h, W, m % mw, m / mw, b, d);
            jpeg_fdct(d);
            jpeg_quantize(d, T, jpeg_table_of(b), zz);
            ac[(size_t)m * 6 + b] = (uint16_t)jpeg_ac_bits(zz, T, jpeg_table_of(b));
        }
    std::vector<uint64_t> off((size_t)n_mcu + 1);
    uint64_t carry = 0;
    for (int m = 0; m < n_mcu; ++m) {                                    // k_jpeg_scan
        int diff[6];
        jpeg_mcu_diffs(coef.data(), m, mw, wb, hb, diff);
        off[m] = carry;
        for (int b = 0; b < 6; ++b) carry += jpeg_dc_bits(diff[b], T, jpeg_table_of(b)) + ac[(size_t)m * 6 + b];
    }
    off[n_mcu] = carry;
    std::vector<uint32_t> words((carry + 31) / 32 + 1, 0);
    if (carry & 7) {
        const int nb = 8 - (int)(carry & 7), at = (int)(carry & 31);
        words[carry >> 5] |= ((1u << nb) - 1) << (32 - at - nb);
    }
    for (int m = n_mcu - 1; m >= 0; --m) {                               // k_jpeg_pack, in an order of its own
        int diff[6];
        jpeg_mcu_diffs(coef.data(), m, mw, wb, hb, diff);
        JpegBitWriter bw;
        jpeg_bw_init(&bw, words.data(), off[m]);
        for (int b = 0; b < 6; ++b) jpeg_put_block(&bw, &coef[((size_t)m * 6 + b) * 64], diff[b], T, jpeg_table_of(b));
        jpeg_bw_flush(&bw);
    }
    const uint64_t nbytes = (carry + 7) / 8;                             // k_jpeg_emit
    const uint64_t len = JPEG_HEADER_BYTES + nbytes + jpeg_count_ff(words.data(), 0, nbytes) + JPEG_EOI_BYTES;
    if (len > cap) return -1;
    jpeg_build_header(W, tile_h, quality, out);
    hc_stuff(words.data(), nbytes, 16, out + JPEG_HEADER_BYTES);
    out[len - 2] = 0xFF;
    out[len - 1] = 0xD9;
    return (int64_t)len;
}
}
