// Device-side prepare_scene: see bvh_build.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace rayb200 {

// Everything prepare_scene leaves resident in HBM, carved out of ONE stream-ordered allocation.
struct DeviceBvh {
  unsigned char *block = nullptr;
  size_t block_bytes = 0;
  int32_t n = 0;
  // packed BVH2C layout walked by the render kernels (scene_host.h)
  float4 *nodes = nullptr, *nodes_soa = nullptr, *geom = nullptr, *colour = nullptr;
  // the LBVH in the reference's own node order (kept for introspection / tests)
  uint32_t *morton = nullptr;
  int32_t *perm = nullptr, *left = nullptr, *right = nullptr, *parent = nullptr;
  float *boxes = nullptr;
};

struct BvhBuildResult {  // small facts the host needs back
  float root_box[6];
  int32_t max_depth, stale_nodes;
};

size_t device_bvh_bytes(int64_t n);
// Carves `block` (device_bvh_bytes(n) bytes) into the arrays of `out` (used by the host-build upload path too).
void carve_device_bvh(unsigned char *block, int64_t n, DeviceBvh &out);
// Builds the LBVH of the n spheres at d_spheres (n x 7 floats: pos, colour, radius) entirely on the device,
// asynchronously on `stream`.  `refit_sweeps` = trunc(log2f(n)) + 2, computed by the caller with the host
// libm exactly as the reference does (bvh.fut:47).  *d_result is written on the device.
cudaError_t build_bvh_device(const float *d_spheres, int64_t n, int32_t refit_sweeps, DeviceBvh &out, BvhBuildResult *d_result,
                             cudaStream_t stream, int64_t *launches);
// The inverse of the build's sphere packing: writes the n sphere records of `bvh` to d_out (n x 7 floats) in the order
// they were given, sphere[perm[k]] = (geom[k].xyz, colour[k].xyz, geom[k].w), bit for bit.  One launch on `stream`.
cudaError_t gather_spheres_device(const DeviceBvh &bvh, int64_t n, float *d_out, cudaStream_t stream, int64_t *launches);

}  // namespace rayb200
