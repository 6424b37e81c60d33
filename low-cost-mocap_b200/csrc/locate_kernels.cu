// SURVEY.md section 8(f) "next" #3: marker triplets -> drone pose, per frame-set.
//
// Replaces locate_objects (reference computer_code/api/helpers.py:424-480).  The per-frame-set code is
// locate_device.cuh, which the CPU tests compile with g++ (tests/hostcheck/locate_host.cpp).
// The greedy scan is order dependent, so one thread owns one frame-set and walks it sequentially;
// frame-sets are independent.
#include "common.cuh"
#include "locate_device.cuh"

static_assert(MOCAP_MAX_ROOTS <= LOC_MAX_POINTS, "the locator's matched-points set holds LOC_MAX_POINTS points");

__global__ void __launch_bounds__(128)
k_locate_objects(const double* __restrict__ obj, const double* __restrict__ err, const int32_t* __restrict__ n_obj,
                 int n_sets, int RMAX, int max_objects, double* __restrict__ out /*[n_sets][max_objects][5]*/,
                 int32_t* __restrict__ drone_index, int32_t* __restrict__ n_out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    locate_frame_set(obj, err, n_obj, s, RMAX, max_objects, out, drone_index, n_out);
}

int launch_locate(mocap_ctx* ctx, const double* obj, const double* err, const int32_t* n_obj, int n_sets,
                  int max_objects, double* out, int32_t* drone_index, int32_t* n_out) {
    if (n_sets <= 0) return MOCAP_OK;
    k_locate_objects<<<(n_sets + 127) / 128, 128, 0, ctx->stream>>>(obj, err, n_obj, n_sets, ctx->cfg.max_roots, max_objects,
                                                                      out, drone_index, n_out);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}
