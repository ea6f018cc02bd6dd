// Device-side prepare_scene: see bvh_build.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace rayb200 {

struct BvhBuildResult {  // small facts the host needs back
  float root_box[6];
  int32_t max_depth, stale_nodes;
};

// Everything prepare_scene leaves resident in HBM, carved out of ONE stream-ordered allocation.  A scene batch's block
// holds its scenes' arrays one after the other (DESIGN.md §5b), with global node, leaf and sphere indices, and three tables.
struct DeviceBvh {
  unsigned char *block = nullptr;
  size_t block_bytes = 0;
  int32_t n = 0;  // leaves (a batch: of all its scenes)
  // packed BVH2C layout walked by the render kernels (scene_host.h)
  float4 *nodes = nullptr, *nodes_soa = nullptr, *geom = nullptr, *colour = nullptr;
  // the LBVH in the reference's own node order (kept for introspection / tests)
  uint32_t *morton = nullptr;
  int32_t *perm = nullptr, *left = nullptr, *right = nullptr, *parent = nullptr;
  float *boxes = nullptr;
  // scene batch only: each scene's build result, whose root box the render kernel reads ([scenes], 32 bytes each), each
  // scene's camera ([scenes][12] floats, laid out as RenderParams::cam), and where each scene starts ([scenes + 1]:
  // scene b's leaves and records start at scene_off[b], its inner nodes at scene_off[b] - b; scene_off[scenes] = n)
  BvhBuildResult *results = nullptr;
  float *cams = nullptr;
  int32_t *scene_off = nullptr;
};

// Bytes of the block of `scenes` trees over n_leaves spheres in all (n_leaves - scenes inner nodes; `tables`: a scene
// batch's, with its tables)
size_t device_bvh_bytes(int64_t n_leaves, int32_t scenes = 1, bool tables = false);
// Carves `block` (device_bvh_bytes(n_leaves, scenes, tables) bytes) into the arrays of `out` (used by the host-build
// upload path too).
void carve_device_bvh(unsigned char *block, int64_t n_leaves, DeviceBvh &out, int32_t scenes = 1, bool tables = false);
// Builds the LBVHs of `scenes` scenes at d_spheres entirely on the device, asynchronously on `stream`, into a new block.
// Scene b's records (7 floats each: pos, colour, radius) are [off[b], off[b + 1]) (host off[scenes + 1], off[0] = 0, each
// scene >= 2 spheres), and it refits for sweeps[b] = trunc(log2f(n_b)) + 2 sweeps (host [scenes]), computed by the
// caller with the host libm exactly as the reference does (bvh.fut:47).  The host tables are read by copies on `stream`
// and must live until it reaches them.  The build results are written on the device to *d_result (one scene);
// d_result == NULL makes the block a scene batch's (any B >= 1), with its tables, and writes them to out.results.  With
// B > 1, perm holds global sphere indices.
cudaError_t build_bvh_device(const float *d_spheres, int32_t scenes, const int32_t *off, const int32_t *sweeps, DeviceBvh &out,
                             BvhBuildResult *d_result, cudaStream_t stream, int64_t *launches);
// Scene s of a batch (its n spheres starting at leaf off_s) as a block of its own (a new allocation in out), every index
// local to it: the arrays a single-scene build of its spheres makes.  One launch on `stream`.
cudaError_t extract_scene_device(const DeviceBvh &batch, int32_t s, int64_t off_s, int64_t n, DeviceBvh &out, cudaStream_t stream,
                                 int64_t *launches);
// The inverse of the build's sphere packing: writes the n sphere records of `bvh` to d_out (n x 7 floats) in the order
// they were given, sphere[perm[k]] = (geom[k].xyz, colour[k].xyz, geom[k].w), bit for bit.  One launch on `stream`.
cudaError_t gather_spheres_device(const DeviceBvh &bvh, int64_t n, float *d_out, cudaStream_t stream, int64_t *launches);

}  // namespace rayb200
