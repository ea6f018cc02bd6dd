// C ABI, part 6: proximity queries (include/ray_b200.h "proximity queries") - the spheres within a radius of each of the
// caller's balls, nearest first - and nearest-sphere queries ("nearest-sphere queries") - the k nearest spheres within a
// radius that may be +inf - for a prepared scene or every scene of a scene batch.  Validation, the choice between the
// stored records and complete boxes, and the launch, shared by both queries; the kernels are in proximity_kernels.cu.
#include "api_internal.h"

#include <cstddef>

#include "proximity.h"

using namespace rayb200_api;

static_assert(sizeof(struct ray_b200_ball) == 16 && offsetof(struct ray_b200_ball, r) == 12,
              "struct ray_b200_ball is 4 floats: centre, r");
static_assert(sizeof(struct ray_b200_near) == 8 && offsetof(struct ray_b200_near, sphere) == 4,
              "struct ray_b200_near is (float d, int32 sphere)");

namespace rayb200_api {

void free_proximity_scratch(futhark_context *ctx) {
  if (ctx->prox_block) cudaFree(ctx->prox_block);
  ctx->prox_block = nullptr;
  ctx->prox_bytes = 0;
}

}  // namespace rayb200_api

namespace {

// Validates and enqueues one query of p's records on the context's stream (lane 0); the caller holds ctx->mu.  `stale`:
// some box of p is not the union of its children's, so the walk reads complete boxes built into the context's scratch
// first.  Q's balls, k and outputs are the caller's; a scene batch's query also sets Q's scene fields.  `nearest`: the
// nearest-sphere kernel (k in [1, 64], no counts) instead of the proximity kernel.
int enqueue(futhark_context *ctx, const futhark_opaque_prepared_scene *p, bool stale, ProximityQuery Q, bool nearest,
            const char *what) {
  const int k_min = nearest ? 1 : 0;
  if (Q.n < 0 || Q.n > ((int64_t)1 << 30)) { set_error(ctx, "%s: n = %lld is outside [0, 2^30]", what, (long long)Q.n); return 1; }
  if (Q.k < k_min || Q.k > 64) { set_error(ctx, "%s: k = %d is outside [%d, 64]", what, Q.k, k_min); return 1; }
  if (Q.n == 0) return 0;
  if (!Q.balls) { set_error(ctx, "%s: NULL balls buffer", what); return 1; }
  if (Q.k > 0 && !Q.near) { set_error(ctx, "%s: NULL near buffer with k = %d", what, Q.k); return 1; }
  if (Q.k == 0 && !Q.counts) { set_error(ctx, "%s: no output (k = 0 and a NULL counts buffer)", what); return 1; }
  if (!p || !p->dev.nodes || !p->dev.geom || !p->dev.perm) { set_error(ctx, "%s: invalid prepared scene", what); return 1; }
  if (p->max_depth > kStackSize - 1) { set_error(ctx, "%s: BVH depth %d exceeds the traversal stack", what, p->max_depth); return 1; }
  if (Q.k == 0) Q.near = nullptr;
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  futhark_context::Lane &L = ctx->lane(0);
  const int64_t n_inner = n_inner_of(p), n_leaves = n_leaves_of(p);
  Q.nodes = p->dev.nodes;
  Q.geom = p->dev.geom;
  Q.perm = p->dev.perm;
  if (stale) {
    const size_t rec_bytes = ((size_t)n_inner * 4 * sizeof(float4) + 255) & ~(size_t)255;
    const size_t need = rec_bytes + refit_scratch_bytes(n_inner, n_leaves);
    if (!ctx->prox_done) CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->prox_done, cudaEventDisableTiming));
    else CUDA_TRY(ctx, cudaStreamWaitEvent(L.stream, ctx->prox_done, 0));  // the last use may be on another stream
    if (ctx->prox_bytes < need) {
      free_proximity_scratch(ctx);
      CUDA_TRY(ctx, cudaMalloc(&ctx->prox_block, need));
      ctx->prox_bytes = need;
    }
    float4 *recs = reinterpret_cast<float4 *>(ctx->prox_block);
    CUDA_TRY(ctx, refit_complete_boxes(p->dev.nodes, p->dev.geom, n_inner, n_leaves, recs, ctx->prox_block + rec_bytes, L.stream,
                                       &ctx->launches));
    Q.nodes = recs;
  }
  CUDA_TRY(ctx, nearest ? launch_nearest(Q, L.stream, &ctx->launches) : launch_proximity(Q, L.stream, &ctx->launches));
  if (stale) CUDA_TRY(ctx, cudaEventRecord(ctx->prox_done, L.stream));
  return record_scene_use(ctx, p, 0);
}

// A query of every scene of batch b, m balls per scene, as enqueue's
int enqueue_batch(futhark_context *ctx, const ray_b200_scene_batch *b, ProximityQuery Q, int64_t m, bool nearest,
                  const char *what) {
  if (!b || !b->scene.dev.block) { set_error(ctx, "%s: invalid scene batch", what); return 1; }
  const int32_t B = b->scene.scenes;
  if (m < 0) { set_error(ctx, "%s: m = %lld balls per scene is negative", what, (long long)m); return 1; }
  if (m > ((int64_t)1 << 30) / B) { set_error(ctx, "%s: %d scenes of %lld balls exceed 2^30 balls", what, B, (long long)m); return 1; }
  bool stale = false;
  for (const BvhBuildResult &r : b->results) stale = stale || r.stale_nodes > 0;
  Q.n = (int64_t)B * m;
  Q.scene_off = b->scene.dev.scene_off;
  Q.balls_per_scene = m;
  return enqueue(ctx, &b->scene, stale, Q, nearest, what);
}

}  // namespace

extern "C" {

int ray_b200_query_spheres(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           const struct ray_b200_ball *balls_dev, int64_t n, int32_t k, struct ray_b200_near *near_dev,
                           int32_t *counts_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  ProximityQuery Q;
  Q.balls = reinterpret_cast<const float *>(balls_dev);
  Q.n = n;
  Q.k = k;
  Q.near = reinterpret_cast<float *>(near_dev);
  Q.counts = counts_dev;
  return enqueue(ctx, p, p && p->stale_nodes > 0, Q, false, "query_spheres");
}

int ray_b200_scene_batch_query_spheres(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                       const struct ray_b200_ball *balls_dev, int64_t m, int32_t k,
                                       struct ray_b200_near *near_dev, int32_t *counts_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  ProximityQuery Q;
  Q.balls = reinterpret_cast<const float *>(balls_dev);
  Q.k = k;
  Q.near = reinterpret_cast<float *>(near_dev);
  Q.counts = counts_dev;
  return enqueue_batch(ctx, b, Q, m, false, "scene_batch_query_spheres");
}

int ray_b200_query_nearest(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           const struct ray_b200_ball *balls_dev, int64_t n, int32_t k, struct ray_b200_near *near_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  ProximityQuery Q;
  Q.balls = reinterpret_cast<const float *>(balls_dev);
  Q.n = n;
  Q.k = k;
  Q.near = reinterpret_cast<float *>(near_dev);
  return enqueue(ctx, p, p && p->stale_nodes > 0, Q, true, "query_nearest");
}

int ray_b200_scene_batch_query_nearest(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                       const struct ray_b200_ball *balls_dev, int64_t m, int32_t k,
                                       struct ray_b200_near *near_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  ProximityQuery Q;
  Q.balls = reinterpret_cast<const float *>(balls_dev);
  Q.k = k;
  Q.near = reinterpret_cast<float *>(near_dev);
  return enqueue_batch(ctx, b, Q, m, true, "scene_batch_query_nearest");
}

int64_t ray_b200_near_size(void) { return (int64_t)sizeof(struct ray_b200_near); }
int64_t ray_b200_ball_size(void) { return (int64_t)sizeof(struct ray_b200_ball); }

}  // extern "C"
