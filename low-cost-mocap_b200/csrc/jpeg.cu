// Baseline JPEG encoding on the device, byte for byte what cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) gives
// (step code and the libjpeg conventions: jpeg.cuh).  Per group of images, four launches:
//   k_jpeg_blocks  one thread per 8 x 8 block: pixels (tiled layout) -> YCbCr -> h2v2 -> islow DCT -> quantise ->
//                  zigzag; stores the coefficients (int16 [MCU][6][64]) and the block's AC code bits;
//   k_jpeg_scan    one CTA per image: per MCU the DC differences (across MCU boundaries, dummies resolved) and the MCU's
//                  code bits, an exclusive scan over the MCUs in scan order -> each MCU's bit offset; zeroes the
//                  image's words and sets the 1-bits that pad the tail to a byte;
//   k_jpeg_pack    one thread per MCU: its codes at its bit offset, plain stores for the words it owns whole, atomicOr
//                  on the two it may share;
//   k_jpeg_emit    one CTA per image: counts the 0xFF bytes, and if the image fits its stride writes the header, the
//                  entropy data with a 0x00 after each 0xFF (per-thread chunks placed by a scan), EOI and the length;
//                  else the length -1 and nothing else.
// The coefficients are stored rather than recomputed in k_jpeg_pack: recomputing repeats the pixel reads, colour
// conversion and DCT (the bulk of the arithmetic) for 2 bytes per coefficient of scratch, 3 bytes per pixel.
#include "common.cuh"
#include "jpeg.cuh"

#define JPEG_THREADS 128
#define JPEG_CTA 512
#define JPEG_GROUP_SCRATCH ((size_t)256 << 20)   // images per group: as many as fit this much scratch (at least one)

static_assert(sizeof(JpegTables) + JPEG_HEADER_BYTES <= JPEG_CONFIG_BYTES, "JPEG_CONFIG_BYTES holds the tables and the header");
static_assert(sizeof(JpegTables) % 4 == 0, "k_jpeg_* copy the tables to shared memory in words");
static_assert(sizeof(((mocap_ctx*)0)->jpeg_cfg) / sizeof(DeviceBuffer) == MOCAP_JPEG_CONFIGS, "one cache slot per configuration");

struct JpegShape {
    int tiles, tile_w, tile_h, W, mw, mh, wb, hb, n_mcu;
    size_t in_stride;                             // bytes of one input image
    size_t coef_stride, off_stride, word_stride;  // per image: int16 coefficients, uint64 offsets, uint32 words
};

static JpegShape jpeg_shape(int tiles, int tile_w, int tile_h) {
    JpegShape s;
    s.tiles = tiles; s.tile_w = tile_w; s.tile_h = tile_h; s.W = tiles * tile_w;
    s.mw = (s.W + 15) / 16; s.mh = (tile_h + 15) / 16;
    s.wb = (s.W + 7) / 8; s.hb = (tile_h + 7) / 8;
    s.n_mcu = s.mw * s.mh;
    s.in_stride = (size_t)s.W * tile_h * 3;
    s.coef_stride = (size_t)s.n_mcu * 6 * 64;
    s.off_stride = (size_t)s.n_mcu + 1;
    s.word_stride = ((size_t)s.n_mcu * JPEG_MCU_MAX_BITS + 31) / 32 + 1;
    return s;
}

// per image: coefficients, AC bits per block, MCU offsets (+ the total), words; picks how many images share the
// scratch (jpeg_encode's layout sizes it)
static size_t jpeg_image_scratch(const JpegShape& s) {
    return s.coef_stride * 2 + (size_t)s.n_mcu * 6 * 2 + s.off_stride * 8 + s.word_stride * 4 + 64;
}

__device__ __forceinline__ void jpeg_load_tables(const JpegTables* g, JpegTables* sh) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
    uint32_t* dst = reinterpret_cast<uint32_t*>(sh);
    for (int i = threadIdx.x; i < (int)(sizeof(JpegTables) / 4); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

__global__ void __launch_bounds__(JPEG_THREADS)
k_jpeg_blocks(const uint8_t* __restrict__ images, JpegShape s, int n_images, const JpegTables* __restrict__ tables,
              int16_t* __restrict__ coef, uint16_t* __restrict__ ac_bits) {
    __shared__ JpegTables T;
    jpeg_load_tables(tables, &T);
    const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t per = (size_t)s.n_mcu * 6;
    if (id >= per * n_images) return;
    const int i = (int)(id / per), m = (int)((id % per) / 6), b = (int)(id % 6);
    const int mx = m % s.mw, my = m / s.mw;
    int16_t* zz = coef + i * s.coef_stride + ((size_t)m * 6 + b) * 64;
    if (jpeg_is_dummy(b, mx, my, s.wb, s.hb)) {
        for (int k = 0; k < 64; ++k) zz[k] = 0;
        ac_bits[id] = T.ac_len[0][0];
        return;
    }
    int d[64];
    int16_t q[64];
    jpeg_block_samples(images + i * s.in_stride, s.tile_w, s.tile_h, s.W, mx, my, b, d);
    jpeg_fdct(d);
    const int t = jpeg_table_of(b);
    jpeg_quantize(d, T, t, q);
    uint4* dst = reinterpret_cast<uint4*>(zz);
    const uint4* src = reinterpret_cast<const uint4*>(q);
#pragma unroll
    for (int k = 0; k < 8; ++k) dst[k] = src[k];
    ac_bits[id] = (uint16_t)jpeg_ac_bits(q, T, t);
}

// exclusive scan of v over the CTA; *total = the sum
__device__ uint64_t jpeg_block_scan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t warp_sum[JPEG_CTA / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[w] = x;
    __syncthreads();
    uint64_t before = 0, all = 0;
    for (int k = 0; k < JPEG_CTA / 32; ++k) {
        if (k < w) before += warp_sum[k];
        all += warp_sum[k];
    }
    __syncthreads();
    *total = all;
    return before + x - v;
}

__global__ void __launch_bounds__(JPEG_CTA)
k_jpeg_scan(JpegShape s, const JpegTables* __restrict__ tables, const int16_t* __restrict__ coef,
            const uint16_t* __restrict__ ac_bits, uint64_t* __restrict__ offs, uint32_t* __restrict__ words) {
    __shared__ JpegTables T;
    jpeg_load_tables(tables, &T);
    const int i = blockIdx.x;
    const int16_t* c = coef + i * s.coef_stride;
    const uint16_t* ac = ac_bits + (size_t)i * s.n_mcu * 6;
    uint64_t* off = offs + i * s.off_stride;
    uint32_t* wd = words + i * s.word_stride;
    uint64_t carry = 0;
    for (int base = 0; base < s.n_mcu; base += JPEG_CTA) {
        const int m = base + threadIdx.x;
        uint64_t bits = 0;
        if (m < s.n_mcu) {
            int diff[6];
            jpeg_mcu_diffs(c, m, s.mw, s.wb, s.hb, diff);
            for (int b = 0; b < 6; ++b) bits += jpeg_dc_bits(diff[b], T, jpeg_table_of(b)) + ac[(size_t)m * 6 + b];
        }
        uint64_t total;
        const uint64_t ex = jpeg_block_scan(bits, &total);
        if (m < s.n_mcu) off[m] = carry + ex;
        carry += total;
    }
    const uint64_t nw = (carry + 31) / 32;
    for (uint64_t k = threadIdx.x; k < nw; k += JPEG_CTA) wd[k] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        off[s.n_mcu] = carry;
        const int rem = (int)(carry & 7);
        if (rem) {                                    // jchuff.c flush_bits: the last byte is completed with 1-bits
            const int nb = 8 - rem, at = (int)(carry & 31);
            wd[carry >> 5] |= ((1u << nb) - 1) << (32 - at - nb);
        }
    }
}

__global__ void __launch_bounds__(JPEG_THREADS)
k_jpeg_pack(JpegShape s, int n_images, const JpegTables* __restrict__ tables, const int16_t* __restrict__ coef,
            const uint64_t* __restrict__ offs, uint32_t* __restrict__ words) {
    __shared__ JpegTables T;
    jpeg_load_tables(tables, &T);
    const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= (size_t)s.n_mcu * n_images) return;
    const int i = (int)(id / s.n_mcu), m = (int)(id % s.n_mcu);
    const int16_t* c = coef + i * s.coef_stride;
    int diff[6];
    jpeg_mcu_diffs(c, m, s.mw, s.wb, s.hb, diff);
    JpegBitWriter bw;
    jpeg_bw_init(&bw, words + i * s.word_stride, offs[i * s.off_stride + m]);
    for (int b = 0; b < 6; ++b) jpeg_put_block(&bw, c + ((size_t)m * 6 + b) * 64, diff[b], T, jpeg_table_of(b));
    jpeg_bw_flush(&bw);
}

#define JPEG_CHUNK 16                                 // entropy bytes per thread per round of k_jpeg_emit

__global__ void __launch_bounds__(JPEG_CTA)
k_jpeg_emit(JpegShape s, const uint8_t* __restrict__ header, const uint64_t* __restrict__ offs, const uint32_t* __restrict__ words,
            uint8_t* __restrict__ out, uint64_t out_stride, int32_t* __restrict__ out_len) {
    const int i = blockIdx.x;
    const uint32_t* wd = words + i * s.word_stride;
    const uint64_t nbytes = (offs[i * s.off_stride + s.n_mcu] + 7) / 8;
    uint64_t ff = 0;
    for (uint64_t j0 = (uint64_t)threadIdx.x * JPEG_CHUNK; j0 < nbytes; j0 += (uint64_t)JPEG_CTA * JPEG_CHUNK)
        ff += jpeg_count_ff(wd, j0, j0 + JPEG_CHUNK < nbytes ? j0 + JPEG_CHUNK : nbytes);
    uint64_t n_ff;
    jpeg_block_scan(ff, &n_ff);
    const uint64_t len = JPEG_HEADER_BYTES + nbytes + n_ff + JPEG_EOI_BYTES;
    if (len > out_stride || len > 0x7fffffffu) {
        if (threadIdx.x == 0) out_len[i] = -1;
        return;
    }
    uint8_t* o = out + i * out_stride;
    for (int j = threadIdx.x; j < JPEG_HEADER_BYTES; j += JPEG_CTA) o[j] = header[j];
    uint8_t* body = o + JPEG_HEADER_BYTES;
    uint64_t carry = 0;
    for (uint64_t base = 0; base < nbytes; base += (uint64_t)JPEG_CTA * JPEG_CHUNK) {
        const uint64_t j0 = base + (uint64_t)threadIdx.x * JPEG_CHUNK;
        const uint64_t j1 = j0 + JPEG_CHUNK < nbytes ? j0 + JPEG_CHUNK : nbytes;
        const uint64_t cnt = j0 < j1 ? jpeg_count_ff(wd, j0, j1) : 0;
        uint64_t total;
        const uint64_t at = carry + jpeg_block_scan(cnt, &total) + j0;
        if (j0 < j1) jpeg_stuff(wd, j0, j1, body, at);
        carry += total;
    }
    if (threadIdx.x == 0) {
        o[len - 2] = 0xFF;
        o[len - 1] = 0xD9;
        out_len[i] = (int32_t)len;
    }
}

// the device copy of the tables and header of (width, height, quality), built on first use; entries are never
// rewritten while work that reads them may be queued (a full cache is dropped after the stream drains)
static int jpeg_config(mocap_ctx* ctx, int width, int height, int quality, const uint8_t** d_cfg) {
    for (int k = 0; k < ctx->jpeg_cfg_n; ++k)
        if (ctx->jpeg_cfg_key[k][0] == width && ctx->jpeg_cfg_key[k][1] == height && ctx->jpeg_cfg_key[k][2] == quality) {
            *d_cfg = ctx->jpeg_cfg[k].as<uint8_t>();
            return MOCAP_OK;
        }
    if (ctx->jpeg_cfg_n == MOCAP_JPEG_CONFIGS) {
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        for (int k = 0; k < ctx->jpeg_cfg_n; ++k) ctx->jpeg_cfg[k].reset();
        ctx->jpeg_cfg_n = 0;
    }
    uint8_t host[JPEG_CONFIG_BYTES];
    memset(host, 0, sizeof host);
    jpeg_build_tables(quality, reinterpret_cast<JpegTables*>(host));
    jpeg_build_header(width, height, quality, host + sizeof(JpegTables));
    const int k = ctx->jpeg_cfg_n;
    const int st = ctx->jpeg_cfg[k].grow(ctx, JPEG_CONFIG_BYTES, Drain::none);
    if (st) return st;
    uint8_t* d = ctx->jpeg_cfg[k].as<uint8_t>();
    // pageable source: the call returns once the bytes are staged, so `host` may go out of scope
    CUDA_TRY(ctx, cudaMemcpyAsync(d, host, JPEG_CONFIG_BYTES, cudaMemcpyHostToDevice, ctx->stream));
    ctx->jpeg_cfg_n++;
    ctx->jpeg_cfg_key[k][0] = width; ctx->jpeg_cfg_key[k][1] = height; ctx->jpeg_cfg_key[k][2] = quality;
    *d_cfg = d;
    return MOCAP_OK;
}

static int jpeg_check(mocap_ctx* ctx, int n_images, int tiles, int tile_w, int tile_h, int quality, const char* who) {
    if (n_images < 0 || tiles < 1 || tile_w < 1 || tile_h < 1)
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: n_images must be >= 0 and tiles, tile_w, tile_h >= 1", who);
    if ((long long)tiles * tile_w > JPEG_MAX_DIM || tile_h > JPEG_MAX_DIM)
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: %lld x %d pixels; JPEG allows at most %d in each direction", who,
                          (long long)tiles * tile_w, tile_h, JPEG_MAX_DIM);
    if (quality < 1 || quality > 100) return mocap_fail(ctx, MOCAP_EINVAL, "%s: quality %d is not in 1..100", who, quality);
    return MOCAP_OK;
}

int jpeg_encode(mocap_ctx* ctx, const uint8_t* images, int n_images, int tiles, int tile_w, int tile_h, int quality,
                uint8_t* out, uint64_t out_stride, int32_t* out_len) {
    if (n_images == 0) return MOCAP_OK;
    const JpegShape s = jpeg_shape(tiles, tile_w, tile_h);
    const uint8_t* cfg;
    int st = jpeg_config(ctx, s.W, tile_h, quality, &cfg);
    if (st) return st;
    const JpegTables* tables = reinterpret_cast<const JpegTables*>(cfg);
    const uint8_t* header = cfg + sizeof(JpegTables);
    const size_t per = jpeg_image_scratch(s);
    size_t fit = JPEG_GROUP_SCRATCH / per;
    if (fit < 1) fit = 1;
    const int group = fit < (size_t)n_images ? (int)fit : n_images;
    int16_t* coef; uint16_t* ac; uint64_t* offs; uint32_t* words;
    st = grow_carved(ctx, ctx->jpeg_scratch, Drain::stream, [&](Layout& L) {
        coef = L.take<int16_t>(s.coef_stride * group); ac = L.take<uint16_t>((size_t)s.n_mcu * 6 * group);
        offs = L.take<uint64_t>(s.off_stride * group); words = L.take<uint32_t>(s.word_stride * group);
    });
    if (st) return st;
    for (int i0 = 0; i0 < n_images; i0 += group) {
        const int g = n_images - i0 < group ? n_images - i0 : group;
        const size_t nb = (size_t)s.n_mcu * 6 * g, nm = (size_t)s.n_mcu * g;
        k_jpeg_blocks<<<(unsigned)((nb + JPEG_THREADS - 1) / JPEG_THREADS), JPEG_THREADS, 0, ctx->stream>>>(
            images + i0 * s.in_stride, s, g, tables, coef, ac);
        k_jpeg_scan<<<g, JPEG_CTA, 0, ctx->stream>>>(s, tables, coef, ac, offs, words);
        k_jpeg_pack<<<(unsigned)((nm + JPEG_THREADS - 1) / JPEG_THREADS), JPEG_THREADS, 0, ctx->stream>>>(s, g, tables, coef, offs, words);
        k_jpeg_emit<<<g, JPEG_CTA, 0, ctx->stream>>>(s, header, offs, words, out + i0 * out_stride, out_stride, out_len + i0);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 4;
    }
    return MOCAP_OK;
}

extern "C" {

uint64_t mocap_jpeg_bound(int width, int height) {
    if (width < 1 || height < 1 || width > JPEG_MAX_DIM || height > JPEG_MAX_DIM) return 0;
    return jpeg_bound(width, height);
}

int mocap_encode_jpeg_dev(mocap_ctx* ctx, const uint8_t* images, int n_images, int tiles, int tile_w, int tile_h,
                          int quality, uint8_t* out, uint64_t out_stride, int32_t* out_len) {
    if (!ctx) return MOCAP_EINVAL;
    if (!images || !out || !out_len) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_encode_jpeg_dev: bad argument");
    int st = jpeg_check(ctx, n_images, tiles, tile_w, tile_h, quality, "mocap_encode_jpeg_dev");
    if (st) return st;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return jpeg_encode(ctx, images, n_images, tiles, tile_w, tile_h, quality, out, out_stride, out_len);
}

int mocap_live_jpeg_host(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                         uint8_t* frames, void* result, int quality, uint8_t* jpeg, uint64_t jpeg_stride, int32_t* jpeg_len) {
    if (!ctx) return MOCAP_EINVAL;
    int st = live_check(ctx, tr, raw, n_reads, mode, timestamps, result, "mocap_live_jpeg_host");
    if (st) return st;
    if (!jpeg || !jpeg_len) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_live_jpeg_host: bad argument");
    const int C = ctx->cfg.n_cam, S = ctx->cfg.width;
    if ((st = jpeg_check(ctx, n_reads, C, S, S, quality, "mocap_live_jpeg_host")) != MOCAP_OK || n_reads == 0) return st;
    const uint64_t bound = jpeg_bound(C * S, S);
    // rows of the device output: the caller's stride (rounded up) when below the bound; an image that fits the rounded
    // row but not the caller's stride is refused below
    const uint64_t dstride = round_up(jpeg_stride < bound ? jpeg_stride : bound, 16);
    int32_t* d_len;
    uint8_t* d_jpeg;
    st = grow_carved(ctx, ctx->jpeg_out, Drain::stream, [&](Layout& L) {
        d_len = L.take<int32_t>(n_reads);
        d_jpeg = L.take<uint8_t>((size_t)n_reads * dstride);
    });
    if (st) return st;
    // the live chain (live.cu), its frames kept on the device for the encoder
    LiveHostRun run;
    if ((st = live_host_run(ctx, tr, raw, n_reads, mode, timestamps, 1, (size_t)n_reads * 4, &run)) != MOCAP_OK) return st;
    if ((st = jpeg_encode(ctx, run.d_frames, n_reads, C, S, S, quality, d_jpeg, dstride, d_len)) != MOCAP_OK) return st;
    if ((st = live_host_finish(ctx, run, frames, result, d_len, jpeg_len)) != MOCAP_OK) return st;    // synchronisation 1
    uint64_t total = 0;
    for (int r = 0; r < n_reads; ++r) {
        if (jpeg_len[r] < 0 || (uint64_t)jpeg_len[r] > jpeg_stride)
            return mocap_fail(ctx, MOCAP_EINVAL, "mocap_live_jpeg_host: the JPEG of read %d does not fit jpeg_stride %llu bytes",
                              r, (unsigned long long)jpeg_stride);
        total += (uint64_t)jpeg_len[r];
    }
    if ((st = ctx->jpeg_host.grow(ctx, total, Drain::none)) != MOCAP_OK) return st;     // the stream is idle here
    uint8_t* h_jpeg = ctx->jpeg_host.as<uint8_t>();
    uint64_t at = 0;
    for (int r = 0; r < n_reads; ++r) {
        CUDA_TRY(ctx, cudaMemcpyAsync(h_jpeg + at, d_jpeg + (size_t)r * dstride, (size_t)jpeg_len[r], cudaMemcpyDeviceToHost,
                                      ctx->stream));
        at += (uint64_t)jpeg_len[r];
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));                                        // synchronisation 2
    at = 0;
    for (int r = 0; r < n_reads; ++r) {
        memcpy(jpeg + (size_t)r * jpeg_stride, h_jpeg + at, (size_t)jpeg_len[r]);
        at += (uint64_t)jpeg_len[r];
    }
    return MOCAP_OK;
}

}  // extern "C"
