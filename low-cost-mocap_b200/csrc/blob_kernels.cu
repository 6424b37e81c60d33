// S1 on sm_90a: threshold + 8-connected blobs + contour-polygon moments.
//
// Replaces Cameras._find_dot (reference computer_code/api/helpers.py:143-163):
//   grey = cvtColor(img, RGB2GRAY); binary = grey > 51; contours = findContours(RETR_TREE,
//   CHAIN_APPROX_SIMPLE); per contour m = cv.moments(contour); centre = int(m10/m00), int(m01/m00)
//   when m00 != 0.
//
// cv.moments of a traced pixel contour is the Green's-theorem polygon moment of the
// polygon through the boundary pixel CENTRES.  For a solid (hole-free) 8-connected
// component that polygon decomposes exactly over 2x2 blocks of pixel centres
// (SURVEY.md §8(a1), Appendix A.1): with n set corners
//     n == 4 : full unit cell      2*area += 2 ; 6*Mx += 6x+3 ; 6*My += 6y+3
//     n == 3 : half cell triangle  2*area += 1 ; 6*Mx += sum x(corners) ; 6*My += sum y(corners)
// so a00, a10, a01 of cv.moments are the integers A2, SX6, SY6 accumulated here, and
// m00 = A2*0.5, m10 = SX6*(1/6), centre = int(m10/m00) is reproduced bit for bit.
//
// Two kernels:
//   k_threshold_segments  HBM-bound stream: every thread loads 16 pixels with one 128-bit
//        load, thresholds them with 3 SWAR integer ops per 4 pixels and appends the rare
//        non-empty 16-bit segment masks to a per-image list (algorithmic bytes: W*H per image,
//        read exactly once; writes are a few hundred bytes per image).
//   k_blob_reduce         one CTA per image on the sparse list only: bitonic sort (raster
//        order), run extraction, union-find over runs in shared memory, per-run cell moments,
//        ranked output in cv.findContours order (descending raster position of first pixel).
#include "common.cuh"
#include "blob_device.cuh"

// 1-channel stream.  UNROLL independent 128-bit loads per thread are issued before any is used.
template <int UNROLL>
__global__ void __launch_bounds__(256)
k_threshold_segments_c1(const uint4* __restrict__ frames, long long n_seg, int seg_per_image,
                        int max_segments, ThreshConst tc, uint32_t* __restrict__ seg_count,
                        uint32_t* __restrict__ seg_list) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; s < n_seg; s += stride * UNROLL) {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long si = s + stride * u;
            v[u] = (si < n_seg) ? ldg_stream(frames + si) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const uint32_t h0 = swar_gt(v[u].x, tc), h1 = swar_gt(v[u].y, tc);
            const uint32_t h2 = swar_gt(v[u].z, tc), h3 = swar_gt(v[u].w, tc);
            if (((h0 | h1 | h2 | h3) & 0x80808080u) == 0) continue;     // the overwhelmingly common case
            const long long si = s + stride * u;
            if (si >= n_seg) continue;
            const uint32_t m = nibble_of(h0) | (nibble_of(h1) << 4) | (nibble_of(h2) << 8) | (nibble_of(h3) << 12);
            append_segment(seg_count, seg_list, max_segments, si, seg_per_image, m);
        }
    }
}

// 3-channel interleaved stream (the layout _find_dot receives).  grey as cv.cvtColor(RGB2GRAY)
// computes it for 8-bit data: (c0*9798 + c1*19235 + c2*3735 + 16384) >> 15  (verified against cv2 4.13).
// The weights sum to 2^15, so grey <= max(c0, c1, c2): a 16-pixel segment none of whose 48 bytes exceeds
// the threshold cannot hold a pixel above it, and that is decided with the same packed byte test as the
// 1-channel stream (39 integer ops per segment).  Only the rare segments that pass get the per-pixel
// arithmetic, from a second (cache-resident) read, so the streaming loop stays small and keeps
// 3 * UNROLL 128-bit loads in flight per thread.
template <int UNROLL>
__global__ void __launch_bounds__(256)
k_threshold_segments_c3(const uint4* __restrict__ frames, long long n_seg, int seg_per_image,
                        int max_segments, int threshold, ThreshConst tc, uint32_t* __restrict__ seg_count,
                        uint32_t* __restrict__ seg_list) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += stride * UNROLL) {
        uint4 v[UNROLL][3];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long si = s + stride * u;
#pragma unroll
            for (int q = 0; q < 3; ++q) v[u][q] = (si < n_seg) ? ldg_stream(frames + si * 3 + q) : make_uint4(0, 0, 0, 0);
        }
        uint32_t todo = 0;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            bool hit;
            if (tc.use_and) hit = any_above<true>(v[u][0], tc) || any_above<true>(v[u][1], tc) || any_above<true>(v[u][2], tc);
            else hit = any_above<false>(v[u][0], tc) || any_above<false>(v[u][1], tc) || any_above<false>(v[u][2], tc);
            todo |= (hit ? 1u : 0u) << u;
        }
        while (todo) {
            const int u = __ffs(todo) - 1;
            todo &= todo - 1;
            const long long si = s + stride * u;
            if (si >= n_seg) break;
            uint32_t w[12];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const uint4 x = __ldg(frames + si * 3 + q);
                w[4 * q + 0] = x.x; w[4 * q + 1] = x.y; w[4 * q + 2] = x.z; w[4 * q + 3] = x.w;
            }
            uint32_t m = 0;
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                const int o = 3 * p;
                const uint32_t c0 = (w[o >> 2] >> ((o & 3) * 8)) & 0xffu;
                const uint32_t c1 = (w[(o + 1) >> 2] >> (((o + 1) & 3) * 8)) & 0xffu;
                const uint32_t c2 = (w[(o + 2) >> 2] >> (((o + 2) & 3) * 8)) & 0xffu;
                const int grey = (int)((c0 * 9798u + c1 * 19235u + c2 * 3735u + 16384u) >> 15);
                m |= (grey > threshold ? 1u : 0u) << p;
            }
            if (m) append_segment(seg_count, seg_list, max_segments, si, seg_per_image, m);
        }
    }
}

// Sparse reduction, common case: one WARP per image (warp-level synchronisation only).  Images
// with more than WE segments / runs or more than WACC blobs are appended to a worklist for the
// full-size kernel below.  Shared memory per warp is a fixed small slab.
template <int WPB, bool WIDE>
__global__ void __launch_bounds__(WPB * 32)
k_blob_reduce_warp(uint32_t* __restrict__ seg_count, const uint32_t* __restrict__ seg_list, int n_images, int E,
                   int W, int H, int max_blobs, int32_t* __restrict__ blob_xy, int32_t* __restrict__ blob_n,
                   int64_t* __restrict__ blob_mom, int32_t* __restrict__ img_flags,
                   uint32_t* __restrict__ worklist, uint32_t* __restrict__ work_count) {
    __shared__ WarpSlab slabs[WPB];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int img = blockIdx.x * WPB + warp;
    if (img >= n_images) return;
    const unsigned cnt = seg_count[img];
    int32_t* ofl = img_flags ? img_flags + img : nullptr;
    if (cnt == 0) {
        if (lane == 0) { blob_n[img] = 0; if (ofl) *ofl = 0; }
        return;
    }
    bool ok = cnt <= BLOB_WE;
    if (ok) {
        WarpSlab& sl = slabs[warp];
        BlobSmem sm;
        sm.seg = sl.seg; sm.parent = sl.parent; sm.base = sl.base; sm.node_seg = sl.node_seg;
        sm.node_bits = sl.node_bits; sm.rank = sl.rank; sm.acc = sl.acc; sm.wsum = nullptr; sm.hs = nullptr;
        sm.rowfirst = BLOB_ROWFIRST(sl, WIDE); sm.row_cap = WIDE ? 0 : BLOB_ROWS;
        const uint32_t* src = seg_list + (size_t)img * E;
        for (int i = lane; i < (int)cnt; i += 32) sm.seg[i] = src[i];
        __syncwarp();
        ok = blob_reduce<32, true, WIDE>(sm, (int)cnt, BLOB_WE, BLOB_WACC, W, H, max_blobs, blob_xy + (size_t)img * max_blobs * 2,
                                   blob_n + img, blob_mom ? blob_mom + (size_t)img * max_blobs * 4 : nullptr, ofl, 0);
    }
    if (lane == 0) {
        if (ok) seg_count[img] = 0;                             // self-cleaning: ready for the next batch
        else worklist[atomicAdd(work_count, 1u)] = (uint32_t)img;
    }
}

// Full-size reduction for the images the warp kernel deferred: persistent CTAs walk the worklist.
template <int NT, bool WIDE>
__global__ void __launch_bounds__(NT)
k_blob_reduce(uint32_t* __restrict__ seg_count, const uint32_t* __restrict__ seg_list, int E, int W, int H,
              int max_blobs, int32_t* __restrict__ blob_xy, int32_t* __restrict__ blob_n,
              int64_t* __restrict__ blob_mom, int32_t* __restrict__ img_flags,
              const uint32_t* __restrict__ worklist, uint32_t* __restrict__ work_count, uint32_t* __restrict__ done_count,
              int stat_images, unsigned long long* __restrict__ stat_acc, unsigned long long* __restrict__ stat_host,
              unsigned long long* __restrict__ hole_win) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BlobSmem sm = carve_blob_smem(smem_raw, E);
    if (hole_win) sm.hole_win = hole_win + (size_t)blockIdx.x * 4 * hole_wide_words(W, H);     // mocap_set_large_holes
    const unsigned n_work = *work_count;
    for (unsigned w = blockIdx.x; w < n_work; w += gridDim.x) {
        const int img = (int)worklist[w];
        const unsigned cnt = seg_count[img];
        __syncthreads();
        if (threadIdx.x == 0) seg_count[img] = 0;
        int flags = 0;
        int n = (int)cnt;
        if (cnt > (unsigned)E) { flags |= MOCAP_F_SEGMENTS; n = 0; }
        int32_t* ofl = img_flags ? img_flags + img : nullptr;
        if (n == 0) {
            if (threadIdx.x == 0) { blob_n[img] = 0; if (ofl) *ofl = flags; }
            continue;
        }
        const uint32_t* src = seg_list + (size_t)img * E;
        for (int i = threadIdx.x; i < n; i += NT) sm.seg[i] = src[i];
        __syncthreads();
        blob_reduce<NT, false, WIDE>(sm, n, E, MOCAP_ACC_CAP, W, H, max_blobs, blob_xy + (size_t)img * max_blobs * 2, blob_n + img,
                               blob_mom ? blob_mom + (size_t)img * max_blobs * 4 : nullptr, ofl, flags);
        __syncthreads();
    }
    // statistic for the host's choice of pipeline for the NEXT batch: blobs found in this batch (images this very
    // launch is still reducing may be missed: it only steers a heuristic), left in mapped host memory by the last CTA
    if (stat_host) {
        unsigned long long local = 0;
        for (int i = blockIdx.x * NT + threadIdx.x; i < stat_images; i += gridDim.x * NT) local += (unsigned)__ldcg(blob_n + i);
        for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
        if ((threadIdx.x & 31) == 0 && local) atomicAdd(stat_acc, local);
        __syncthreads();
    }
    if (threadIdx.x == 0) {                                     // the last CTA to finish re-arms the worklist
        __threadfence();
        if (atomicAdd(done_count, 1u) == gridDim.x - 1) {
            *work_count = 0; *done_count = 0;
            if (stat_host) {
                __threadfence();
                stat_host[0] = atomicExch(stat_acc, 0ull);
                stat_host[1] = (unsigned long long)stat_images;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------------------------
int launch_detect(mocap_ctx* ctx, const uint8_t* frames, int n_images, int channels, int threshold,
                  int32_t* blob_xy, int32_t* blob_n, int64_t* blob_mom, int32_t* img_flags) {
    const mocap_config& c = ctx->cfg;
    const int seg_per_image = c.width * c.height / MOCAP_SEG_PX;
    const long long n_seg = (long long)n_images * seg_per_image;
    const int E = c.max_segments;
    if (n_images <= 0) return MOCAP_OK;

    int st = timing_begin(ctx);
    if (st) return st;
    const int threads = 256;
    const ThreshConst tc = thresh_const(threshold);
    const long long cap = (long long)ctx->num_sms * 8;      // 8 CTAs of 256 threads fill an SM
    if (channels == 1) {
        constexpr int UNROLL = 8;
        long long want = (n_seg + (long long)threads * UNROLL - 1) / ((long long)threads * UNROLL);
        const int grid = (int)(want < cap ? want : cap);
        k_threshold_segments_c1<UNROLL><<<grid, threads, 0, ctx->stream>>>(
            reinterpret_cast<const uint4*>(frames), n_seg, seg_per_image, E, tc, ctx->d_seg_count, ctx->d_seg_list);
    } else {
        constexpr int UNROLL = 2;
        long long want = (n_seg + (long long)threads * UNROLL - 1) / ((long long)threads * UNROLL);
        const int grid = (int)(want < cap ? want : cap);
        k_threshold_segments_c3<UNROLL><<<grid, threads, 0, ctx->stream>>>(
            reinterpret_cast<const uint4*>(frames), n_seg, seg_per_image, E, threshold, tc, ctx->d_seg_count, ctx->d_seg_list);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    if ((st = timing_end(ctx)) != MOCAP_OK) return st;
    constexpr int WPB = 8;
    if (moments_wide(c))
        k_blob_reduce_warp<WPB, true><<<(n_images + WPB - 1) / WPB, WPB * 32, 0, ctx->stream>>>(
            ctx->d_seg_count, ctx->d_seg_list, n_images, E, c.width, c.height, c.max_blobs, blob_xy, blob_n, blob_mom, img_flags,
            ctx->d_worklist, ctx->d_work_count);
    else
        k_blob_reduce_warp<WPB, false><<<(n_images + WPB - 1) / WPB, WPB * 32, 0, ctx->stream>>>(
            ctx->d_seg_count, ctx->d_seg_list, n_images, E, c.width, c.height, c.max_blobs, blob_xy, blob_n, blob_mom, img_flags,
            ctx->d_worklist, ctx->d_work_count);
    CUDA_TRY(ctx, cudaGetLastError());
    if ((st = launch_blob_fallback(ctx, blob_xy, blob_n, blob_mom, img_flags, n_images)) != MOCAP_OK) return st;
    ctx->launches += 2;      // stream kernel + warp-level reduce (the fallback counted itself)
    return MOCAP_OK;
}

// full-size reduction of the images on the worklist (exits at once when the list is empty)
int launch_blob_fallback(mocap_ctx* ctx, int32_t* blob_xy, int32_t* blob_n, int64_t* blob_mom, int32_t* img_flags, int n_images) {
    const mocap_config& c = ctx->cfg;
    constexpr int NT = 128;
    const int E = c.max_segments;
    const size_t smem = blob_reduce_smem_bytes(E);
    const int grid2 = ctx->num_sms;
    if (moments_wide(c))
        k_blob_reduce<NT, true><<<grid2, NT, smem, ctx->stream>>>(ctx->d_seg_count, ctx->d_seg_list, E, c.width, c.height,
                                                               c.max_blobs, blob_xy, blob_n, blob_mom, img_flags,
                                                               ctx->d_worklist, ctx->d_work_count, ctx->d_work_count + 1,
                                                               n_images, ctx->stat_acc.as<unsigned long long>(), ctx->pipeline_auto ? ctx->d_stat_host : nullptr,
                                                               ctx->hole_win.as<unsigned long long>());
    else
        k_blob_reduce<NT, false><<<grid2, NT, smem, ctx->stream>>>(ctx->d_seg_count, ctx->d_seg_list, E, c.width, c.height,
                                                                c.max_blobs, blob_xy, blob_n, blob_mom, img_flags,
                                                                ctx->d_worklist, ctx->d_work_count, ctx->d_work_count + 1,
                                                               n_images, ctx->stat_acc.as<unsigned long long>(), ctx->pipeline_auto ? ctx->d_stat_host : nullptr,
                                                               ctx->hole_win.as<unsigned long long>());
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}

int timing_begin(mocap_ctx* ctx) {
    if (!ctx->timing_on) return MOCAP_OK;
    if (ctx->tim_used == 64) { const int st = timing_flush(ctx); if (st) return st; }
    CUDA_TRY(ctx, cudaEventRecord(ctx->tim_ev[2 * ctx->tim_used], ctx->stream));
    return MOCAP_OK;
}

int timing_end(mocap_ctx* ctx) {
    if (!ctx->timing_on) return MOCAP_OK;
    CUDA_TRY(ctx, cudaEventRecord(ctx->tim_ev[2 * ctx->tim_used + 1], ctx->stream));
    ctx->tim_used += 1;
    return MOCAP_OK;
}

int timing_flush(mocap_ctx* ctx) {
    for (int i = 0; i < ctx->tim_used; ++i) {
        float ms = 0.f;
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->tim_ev[2 * i + 1]));
        CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->tim_ev[2 * i], ctx->tim_ev[2 * i + 1]));
        ctx->detect_ms_sum += ms;
        ctx->detect_ms_n += 1;
    }
    ctx->tim_used = 0;
    return MOCAP_OK;
}

// the whole-image window of the RETR_TREE slow path, one per CTA of k_blob_reduce (grid = num_sms): on = allocate, off = free
int blob_set_large_holes(mocap_ctx* ctx, int on) {
    if (!on == !ctx->hole_win.get()) return MOCAP_OK;
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));          // a k_blob_reduce in flight may still use the scratch
    if (!on) {
        ctx->hole_win.reset();
        return MOCAP_OK;
    }
    const size_t bytes = (size_t)ctx->num_sms * 4 * hole_wide_words(ctx->cfg.width, ctx->cfg.height) * sizeof(unsigned long long);
    if (ctx->hole_win.grow(ctx, bytes, Drain::none) != MOCAP_OK)
        return mocap_fail(ctx, MOCAP_ENOMEM, "mocap_set_large_holes: %zu bytes of device memory for the whole-image windows", bytes);
    return MOCAP_OK;
}

int blob_kernels_init(mocap_ctx* ctx) {
    const size_t smem = blob_reduce_smem_bytes(ctx->cfg.max_segments);
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_blob_reduce<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_blob_reduce<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return MOCAP_OK;
}
