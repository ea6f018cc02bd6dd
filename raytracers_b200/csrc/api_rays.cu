// C ABI, part 5: ray queries (include/ray_b200.h "ray queries") - caller-supplied rays traced against a prepared scene
// by the warp-queue kernel in ray mode (render_kernels.cu), either to their closest hit (objs_hit), along their whole
// path (ray_colour) (both Query::kClosest), to their first accepted sphere (occlusion, Query::kAnyHit), or to the k
// nearest of their accepted spheres (multi-hit, Query::kMultiHit).  The last three also come in a ranged form whose rays
// carry their own intervals (struct ray_b200_ray).  Each has a scene-batch form (ray_b200_scene_batch_trace_*): m rays per
// scene of a batch, traced by the same kernel in one launch (Query::kBatchClosest / kBatchAnyHit / kBatchMultiHit).
#include "api_internal.h"

#include <cmath>
#include <cstddef>

using namespace rayb200_api;

static_assert(sizeof(struct ray_b200_hit) == 32, "struct ray_b200_hit is 32 bytes");
static_assert(sizeof(struct ray_b200_ray) == 32 && offsetof(struct ray_b200_ray, t_min) == 12 &&
                  offsetof(struct ray_b200_ray, d) == 16 && offsetof(struct ray_b200_ray, t_max) == 28,
              "struct ray_b200_ray is 8 floats: origin, t_min, direction, t_max");

namespace {

// Validates, plans and enqueues one query of kind `kind` on the context's stream (lane 0); the caller holds ctx->mu.  The
// entry point fills the fields of Q its query uses (rays, interval, depth limit, output buffers); out is the output buffer
// the query needs.  `ranged`: the rays are struct ray_b200_ray[n], each with its own interval, which the host cannot check
// without a device sync; the kernel gives an invalid one the empty answer instead.  A scene batch's query (kind
// is_batch_ray) passes the batch's scene, with n = B m and Q's batch fields set by trace_batch.
int enqueue(futhark_context *ctx, const futhark_opaque_prepared_scene *p, int64_t n, Query kind, bool ranged, RayQuery Q,
            const void *out, const char *what) {
  if (n < 0 || n > ((int64_t)1 << 30)) { set_error(ctx, "%s: n = %lld is outside [0, 2^30]", what, (long long)n); return 1; }
  if (!ranged && (!std::isfinite(Q.t_min) || !std::isfinite(Q.t_max) || Q.t_min < 0.0f)) {
    set_error(ctx, "%s: the interval (%g, %g) needs a finite t_min >= 0 and a finite t_max", what, (double)Q.t_min,
              (double)Q.t_max);
    return 1;
  }
  if (Q.max_depth < 0 || Q.max_depth > 65535) { set_error(ctx, "%s: max_depth %d is outside [0, 65535]", what, Q.max_depth); return 1; }
  if (single_scene_kind(kind) == Query::kMultiHit && (Q.k < 1 || Q.k > 64)) { set_error(ctx, "%s: k = %d is outside [1, 64]", what, Q.k); return 1; }
  if (n == 0) return 0;
  if (!Q.rays || !out) { set_error(ctx, "%s: NULL device buffer", what); return 1; }
  if (!p || !p->dev.nodes || !p->dev.perm) { set_error(ctx, "%s: invalid prepared scene", what); return 1; }
  if (p->max_depth > kStackSize - 1) { set_error(ctx, "%s: BVH depth %d exceeds the traversal stack", what, p->max_depth); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  futhark_context::Lane &L = ctx->lane(0);
  CUDA_TRY(ctx, cudaEventRecord(ctx->ev_start, L.stream));
  if (Q.max_depth == 0) {  // a path query whose ray_colour loop does not run: colour 0, no objs_hit call
    CUDA_TRY(ctx, cudaMemsetAsync(Q.rgb, 0, (size_t)n * 3 * sizeof(float), L.stream));
    if (Q.segments) CUDA_TRY(ctx, cudaMemsetAsync(Q.segments, 0, (size_t)n * sizeof(int32_t), L.stream));
  } else {
    RenderParams P;
    LaunchConfig lc;
    fill_scene_params(p, P);
    if (plan_warpqueue(ctx, p, false, false, true, what, P, lc)) return 1;
    P.work_cursor = L.work_cursor;
    Q.perm = p->dev.perm;
    Q.n = (int32_t)n;
    CUDA_TRY(ctx, cudaMemsetAsync(L.work_cursor, 0, 2 * sizeof(int32_t), L.stream));
    CUDA_TRY(ctx, launch_warpqueue(P, kind, ranged, Q, lc, L.stream, &ctx->launches));
    CUDA_TRY(ctx, cudaGetLastError());
    record_plan(ctx, P, lc, kind, ranged, Q);
  }
  if (record_scene_use(ctx, p, 0)) return 1;
  CUDA_TRY(ctx, cudaEventRecord(ctx->ev_stop, L.stream));
  ctx->have_timing = true;
  return 0;
}

// A query of one prepared scene
int trace(futhark_context *ctx, const futhark_opaque_prepared_scene *p, int64_t n, Query kind, bool ranged, RayQuery Q,
          const void *out, const char *what) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  return enqueue(ctx, p, n, kind, ranged, Q, out, what);
}

// A query of scene batch b, m rays per scene (include/ray_b200.h "scene batches"): the single-scene query of kind `kind`
// as one launch over the B m rays, each traced in its own scene's tree (root node scene_off[b] - b and root box b of
// the batch's device tables, as the batch render reads them), planned over all B trees as the batch render is
int trace_batch(futhark_context *ctx, const ray_b200_scene_batch *b, int64_t m, Query kind, bool ranged, RayQuery Q,
                const void *out, const char *what) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!b || !b->scene.dev.block) { set_error(ctx, "%s: invalid scene batch", what); return 1; }
  const int32_t B = b->scene.scenes;
  if (m < 0) { set_error(ctx, "%s: m = %lld rays per scene is negative", what, (long long)m); return 1; }
  if (m > ((int64_t)1 << 30) / B) {
    set_error(ctx, "%s: %d scenes of %lld rays exceed 2^30 rays", what, B, (long long)m);
    return 1;
  }
  Q.root_boxes = reinterpret_cast<const float *>(b->scene.dev.results);
  Q.scene_off = b->scene.dev.scene_off;
  Q.rays_per_scene = (int32_t)m;
  return enqueue(ctx, &b->scene, (int64_t)B * m, kind, ranged, Q, out, what);
}

// The rays and interval of a query of one segment (max_depth 1; a ranged query's interval is each ray's own)
RayQuery one_segment(const float *rays, float t_min, float t_max) {
  RayQuery Q{};
  Q.rays = rays;
  Q.t_min = t_min;
  Q.t_max = t_max;
  Q.max_depth = 1;
  return Q;
}

}  // namespace

extern "C" {

int ray_b200_trace_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev, int64_t n,
                        float t_min, float t_max, struct ray_b200_hit *hits_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.hits = reinterpret_cast<float *>(hits_dev);
  return trace(ctx, p, n, Query::kClosest, false, Q, hits_dev, "trace_hits");
}

int ray_b200_trace_paths(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev, int64_t n,
                         int32_t max_depth, float *rgb_dev, int32_t *segments_dev) {
  RayQuery Q{};
  Q.rays = rays_dev;
  Q.t_min = 0.0f;            // ray_colour calls objs_hit with (0, 1e9) (ray.fut:130)
  Q.t_max = 1000000000.0f;
  Q.max_depth = max_depth;
  Q.rgb = rgb_dev;
  Q.segments = segments_dev;
  return trace(ctx, p, n, Query::kClosest, false, Q, rgb_dev, "trace_paths");
}

int ray_b200_trace_occluded(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev,
                            int64_t n, float t_min, float t_max, uint8_t *occluded_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.occluded = occluded_dev;
  return trace(ctx, p, n, Query::kAnyHit, false, Q, occluded_dev, "trace_occluded");
}

int ray_b200_trace_multi_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev,
                              int64_t n, float t_min, float t_max, int32_t k, struct ray_b200_hit *hits_dev, int32_t *counts_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.k = k;
  Q.hits = reinterpret_cast<float *>(hits_dev);
  Q.counts = counts_dev;
  return trace(ctx, p, n, Query::kMultiHit, false, Q, hits_dev, "trace_multi_hits");
}

int ray_b200_trace_hits_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                               const struct ray_b200_ray *rays_dev, int64_t n, struct ray_b200_hit *hits_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.hits = reinterpret_cast<float *>(hits_dev);
  return trace(ctx, p, n, Query::kClosest, true, Q, hits_dev, "trace_hits_ranged");
}

int ray_b200_trace_occluded_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                                   const struct ray_b200_ray *rays_dev, int64_t n, uint8_t *occluded_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.occluded = occluded_dev;
  return trace(ctx, p, n, Query::kAnyHit, true, Q, occluded_dev, "trace_occluded_ranged");
}

int ray_b200_trace_multi_hits_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                                     const struct ray_b200_ray *rays_dev, int64_t n, int32_t k,
                                     struct ray_b200_hit *hits_dev, int32_t *counts_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.k = k;
  Q.hits = reinterpret_cast<float *>(hits_dev);
  Q.counts = counts_dev;
  return trace(ctx, p, n, Query::kMultiHit, true, Q, hits_dev, "trace_multi_hits_ranged");
}

int ray_b200_scene_batch_trace_hits(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                    int64_t m, float t_min, float t_max, struct ray_b200_hit *hits_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.hits = reinterpret_cast<float *>(hits_dev);
  return trace_batch(ctx, b, m, Query::kBatchClosest, false, Q, hits_dev, "scene_batch_trace_hits");
}

int ray_b200_scene_batch_trace_paths(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                     int64_t m, int32_t max_depth, float *rgb_dev, int32_t *segments_dev) {
  RayQuery Q{};
  Q.rays = rays_dev;
  Q.t_min = 0.0f;            // as ray_b200_trace_paths
  Q.t_max = 1000000000.0f;
  Q.max_depth = max_depth;
  Q.rgb = rgb_dev;
  Q.segments = segments_dev;
  return trace_batch(ctx, b, m, Query::kBatchClosest, false, Q, rgb_dev, "scene_batch_trace_paths");
}

int ray_b200_scene_batch_trace_occluded(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                        int64_t m, float t_min, float t_max, uint8_t *occluded_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.occluded = occluded_dev;
  return trace_batch(ctx, b, m, Query::kBatchAnyHit, false, Q, occluded_dev, "scene_batch_trace_occluded");
}

int ray_b200_scene_batch_trace_multi_hits(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                          const float *rays_dev, int64_t m, float t_min, float t_max, int32_t k,
                                          struct ray_b200_hit *hits_dev, int32_t *counts_dev) {
  RayQuery Q = one_segment(rays_dev, t_min, t_max);
  Q.k = k;
  Q.hits = reinterpret_cast<float *>(hits_dev);
  Q.counts = counts_dev;
  return trace_batch(ctx, b, m, Query::kBatchMultiHit, false, Q, hits_dev, "scene_batch_trace_multi_hits");
}

int ray_b200_scene_batch_trace_hits_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                           const struct ray_b200_ray *rays_dev, int64_t m, struct ray_b200_hit *hits_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.hits = reinterpret_cast<float *>(hits_dev);
  return trace_batch(ctx, b, m, Query::kBatchClosest, true, Q, hits_dev, "scene_batch_trace_hits_ranged");
}

int ray_b200_scene_batch_trace_occluded_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                               const struct ray_b200_ray *rays_dev, int64_t m, uint8_t *occluded_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.occluded = occluded_dev;
  return trace_batch(ctx, b, m, Query::kBatchAnyHit, true, Q, occluded_dev, "scene_batch_trace_occluded_ranged");
}

int ray_b200_scene_batch_trace_multi_hits_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                                 const struct ray_b200_ray *rays_dev, int64_t m, int32_t k,
                                                 struct ray_b200_hit *hits_dev, int32_t *counts_dev) {
  RayQuery Q = one_segment(reinterpret_cast<const float *>(rays_dev), 0.0f, 0.0f);
  Q.k = k;
  Q.hits = reinterpret_cast<float *>(hits_dev);
  Q.counts = counts_dev;
  return trace_batch(ctx, b, m, Query::kBatchMultiHit, true, Q, hits_dev, "scene_batch_trace_multi_hits_ranged");
}

int64_t ray_b200_hit_size(void) { return (int64_t)sizeof(struct ray_b200_hit); }
int64_t ray_b200_ray_size(void) { return (int64_t)sizeof(struct ray_b200_ray); }

}  // extern "C"
