// Test-only host build of csrc/locate_device.cuh (the marker-triplet drone locator), so that the locator can be checked
// against the oracle on a machine without a GPU.  It walks a batch the way k_locate_objects does, one frame-set after
// another.  NOT part of libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include "../../low-cost-mocap_b200/csrc/locate_device.cuh"

extern "C" {
// the arguments of mocap_locate_objects_dev, host arrays, with the context's max_roots spelled out
void hc_locate(const double* obj, const double* err, const int32_t* n_obj, int n_sets, int max_roots, int max_objects,
               double* objects, int32_t* drone_index, int32_t* n_objects) {
    for (int s = 0; s < n_sets; ++s) locate_frame_set(obj, err, n_obj, s, max_roots, max_objects, objects, drone_index, n_objects);
}
}
