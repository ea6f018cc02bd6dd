// Proximity queries (include/ray_b200.h "proximity queries"): the kernels of proximity_kernels.cu as the host path
// (api_proximity.cu) launches them.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace rayb200 {

// One launch of the query kernel: n balls against the BVH2C records `nodes` (the prepared scene's, or complete boxes
// built by refit_complete_boxes in the same layout) and the Morton-ordered sphere records `geom`.
struct ProximityQuery {
  const float4 *nodes = nullptr;
  const float4 *geom = nullptr;
  const int32_t *perm = nullptr;     // Morton-sorted leaf -> caller index (global in a scene batch)
  const float *balls = nullptr;      // [n][4]: centre.xyz, r (4-byte aligned)
  int64_t n = 0;
  int32_t k = 0;                     // records per ball, [0, 64] ([1, 64] for the nearest-sphere kernel)
  float *near = nullptr;             // [n][k] struct ray_b200_near (d, sphere); NULL when k == 0
  int32_t *counts = nullptr;         // [n] or NULL (always NULL for the nearest-sphere kernel)
  // scene batch: ball i belongs to scene i / balls_per_scene, whose root record is scene_off[b] - b and whose spheres
  // are numbered from scene_off[b]; NULL for one scene (root record 0, spheres from 0)
  const int32_t *scene_off = nullptr;
  int64_t balls_per_scene = 0;
};

// Scratch of refit_complete_boxes for n_inner records and n_leaves leaves, in bytes
size_t refit_scratch_bytes(int64_t n_inner, int64_t n_leaves);
// Copies the n_inner records at `nodes` to `out` and replaces every inner child's box by the union of its subtree's
// sphere boxes (c - r, c + r per axis, joined by fminf / fmaxf), bottom-up: the refit of the fixed sweep count run to its
// fixpoint.  Leaf children keep their always-pass boxes and every child pointer is copied.  Roots are the records no
// record points to (one per scene of a batch).  `scratch`: refit_scratch_bytes(n_inner, n_leaves) bytes.  A copy, two
// memsets and two launches on `stream`.
cudaError_t refit_complete_boxes(const float4 *nodes, const float4 *geom, int64_t n_inner, int64_t n_leaves, float4 *out,
                                 void *scratch, cudaStream_t stream, int64_t *launches);
// One launch of the query kernel on `stream`, with the register bucket that holds Q.k records
cudaError_t launch_proximity(const ProximityQuery &Q, cudaStream_t stream, int64_t *launches);
// One launch of the nearest-sphere kernel on `stream` (include/ray_b200.h "nearest-sphere queries"): the Q.k nearest
// spheres within each ball, r = +inf allowed, Q.k in [1, 64]; Q.counts is not written
cudaError_t launch_nearest(const ProximityQuery &Q, cudaStream_t stream, int64_t *launches);

}  // namespace rayb200
