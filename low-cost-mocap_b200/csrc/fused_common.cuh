// Pieces of the single-pass pipeline kernel (fused_device.cuh, launched by fused_kernel.cu): its parameters and
// the "last arriver" follow-up work.
#pragma once
#include "common.cuh"
#include "blob_device.cuh"
#include "match_device.cuh"

struct FusedParams {
    const uint4* frames;
    long long total_units;
    int n_sets, C, W, H;
    int seg_per_image, units_per_image, iters_per_unit;
    int u4_per_image;              // 128-bit words per image: seg_per_image (1 channel) or 3 * seg_per_image (H x W x 3 interleaved)
    int threshold;                 // the raw threshold (the 3-channel path compares the grey value with it)
    ThreshConst tc;
    int E;                         // stride of the global segment lists
    uint32_t* seg_count; uint32_t* seg_list;
    uint32_t* img_done;            // [n_images]  finished units per image (self-resetting)
    uint32_t* set_done;            // [n_sets]    finished images per frame-set (self-resetting)
    uint32_t* set_defer;           // [n_sets]    != 0: an image of the set went to the worklist
    unsigned long long* unit_counter;
    int32_t* blob_xy; int32_t* blob_n; int32_t* img_flags;
    uint32_t* img_worklist; uint32_t* img_work_count;
    uint32_t* set_worklist; uint32_t* set_work_count;
    const CameraTables* tb;
    int MB, RMAX, KC; uint32_t GMAX;
    double* obj; double* err; int32_t* n_obj; int32_t* set_flags;
    int32_t* track_xy;             // optional: pixel of every winner per camera (mocap_pipeline_tracks_dev)
    size_t slab_bytes;
};

// The follow-up work of the warp that completed the LAST slice of image `img`: reduce the image's segment
// list to blobs (warp-level), and -- if that was the last image of its frame-set -- run the matcher.
template <bool WIDE>
__device__ __forceinline__ void finish_image(const FusedParams& P, unsigned char* slab, int img, int lane) {
    // ---- this warp finished the image: reduce its segment list to blobs ----------------------
    __threadfence();                                   // acquire: everybody else's list entries
    const unsigned cnt = __ldcg(&P.seg_count[img]);
    bool deferred = false;
    if (cnt == 0) {
        if (lane == 0) { P.blob_n[img] = 0; if (P.img_flags) P.img_flags[img] = 0; }
    } else {
        bool ok = cnt <= BLOB_WE;
        if (ok) {
            WarpSlab& sl = *reinterpret_cast<WarpSlab*>(slab);
            BlobSmem sm;
            sm.seg = sl.seg; sm.parent = sl.parent; sm.base = sl.base; sm.node_seg = sl.node_seg;
            sm.node_bits = sl.node_bits; sm.rank = sl.rank; sm.acc = sl.acc; sm.wsum = nullptr; sm.hs = nullptr;
    sm.rowfirst = BLOB_ROWFIRST(sl, WIDE); sm.row_cap = WIDE ? 0 : BLOB_ROWS;
            const uint32_t* lst = P.seg_list + (size_t)img * P.E;
            for (int i = lane; i < (int)cnt; i += 32) sm.seg[i] = __ldcg(lst + i);
            __syncwarp();
            ok = blob_reduce<32, true, WIDE>(sm, (int)cnt, BLOB_WE, BLOB_WACC, P.W, P.H, P.MB,
                                             P.blob_xy + (size_t)img * P.MB * 2, P.blob_n + img, nullptr,
                                             P.img_flags ? P.img_flags + img : nullptr, 0);
            __syncwarp();
        }
        if (lane == 0) {
            if (ok) P.seg_count[img] = 0;             // self-cleaning
            else P.img_worklist[atomicAdd(P.img_work_count, 1u)] = (uint32_t)img;
        }
        deferred = !ok;
    }
    if (lane == 0) { P.img_done[img] = 0; }
    const int set = img / P.C;
    if (deferred && lane == 0) atomicOr(&P.set_defer[set], 1u);
    __threadfence();                                   // release: blob list of this image
    __syncwarp();
    unsigned sd = 0;
    if (lane == 0) {
        __threadfence();                               // publishing lane: fence after the warp barrier, then the counter
        sd = atomicAdd(&P.set_done[set], 1u);
    }
    sd = __shfl_sync(0xffffffffu, sd, 0);
    if (sd != (unsigned)P.C - 1) return;

    // ---- this warp finished the frame-set: match + triangulate --------------------------------
    __threadfence();                                   // acquire: blob lists of the other cameras
    const unsigned defer = __ldcg(&P.set_defer[set]);
    __syncwarp();                                      // every lane has read the mark before lane 0 clears it
    if (lane == 0) { P.set_done[set] = 0; P.set_defer[set] = 0; }
    if (defer) {
        if (lane == 0) P.set_worklist[atomicAdd(P.set_work_count, 1u)] = (uint32_t)set;
        return;
    }
    WarpState ws = carve_warp_state(slab, P.RMAX, P.C, P.KC, P.MB);
    match_triangulate_warp(P.tb, ws, P.blob_xy + (size_t)set * P.C * P.MB * 2, P.blob_n + (size_t)set * P.C, set, lane,
                           P.C, P.MB, P.RMAX, P.KC, P.GMAX, P.obj, P.err, P.n_obj, P.set_flags, nullptr, P.track_xy,
                           P.img_flags ? P.img_flags + (size_t)set * P.C : nullptr);
    __syncwarp();
}

