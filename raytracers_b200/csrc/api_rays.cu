// C ABI, part 5: ray queries (include/ray_b200.h "ray queries") - caller-supplied rays traced against a prepared scene
// by the warp-queue kernel in ray mode (render_kernels.cu), either to their closest hit (objs_hit), along their whole
// path (ray_colour), to their first accepted sphere (occlusion, the any-hit instantiations), or to the k nearest of
// their accepted spheres (multi-hit, the multi-hit instantiations).
#include "api_internal.h"

#include <cmath>

using namespace rayb200_api;

static_assert(sizeof(struct ray_b200_hit) == 32, "struct ray_b200_hit is 32 bytes");

namespace {

// Validates, plans and enqueues one query on the context's stream (lane 0).  multi: multi-hit query of k records per ray
// into hits (and counts, optional), else hits != NULL: hit query, occluded != NULL: occlusion query, else path query.
int trace(futhark_context *ctx, const futhark_opaque_prepared_scene *p, const float *rays, int64_t n, float t_min, float t_max,
          int32_t max_depth, ray_b200_hit *hits, float *rgb, int32_t *segments, uint8_t *occluded, bool multi, int32_t k,
          int32_t *counts, const char *what) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (n < 0 || n > ((int64_t)1 << 30)) { set_error(ctx, "%s: n = %lld is outside [0, 2^30]", what, (long long)n); return 1; }
  if (!std::isfinite(t_min) || !std::isfinite(t_max) || t_min < 0.0f) {
    set_error(ctx, "%s: the interval (%g, %g) needs a finite t_min >= 0 and a finite t_max", what, (double)t_min, (double)t_max);
    return 1;
  }
  if (max_depth < 0 || max_depth > 65535) { set_error(ctx, "%s: max_depth %d is outside [0, 65535]", what, max_depth); return 1; }
  if (multi && (k < 1 || k > 64)) { set_error(ctx, "%s: k = %d is outside [1, 64]", what, k); return 1; }
  if (n == 0) return 0;
  if (!rays || (!hits && !rgb && !occluded)) { set_error(ctx, "%s: NULL device buffer", what); return 1; }
  if (!p || !p->dev.nodes || !p->dev.perm) { set_error(ctx, "%s: invalid prepared scene", what); return 1; }
  if (p->max_depth > kStackSize - 1) { set_error(ctx, "%s: BVH depth %d exceeds the traversal stack", what, p->max_depth); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  futhark_context::Lane &L = ctx->lanes[0];
  L.stream = ctx->stream;
  CUDA_TRY(ctx, cudaEventRecord(ctx->ev_start, L.stream));
  if (!hits && !occluded && max_depth == 0) {  // ray_colour's loop does not run: colour 0, no objs_hit call
    CUDA_TRY(ctx, cudaMemsetAsync(rgb, 0, (size_t)n * 3 * sizeof(float), L.stream));
    if (segments) CUDA_TRY(ctx, cudaMemsetAsync(segments, 0, (size_t)n * sizeof(int32_t), L.stream));
  } else {
    RenderParams P;
    LaunchConfig lc;
    fill_scene_params(p, P);
    if (plan_warpqueue(ctx, p, false, false, true, what, P, lc)) return 1;
    P.work_cursor = L.work_cursor;
    RayQuery Q;
    Q.rays = rays;
    Q.rgb = rgb;
    Q.segments = segments;
    Q.hits = reinterpret_cast<float *>(hits);
    Q.perm = p->dev.perm;
    Q.n = (int32_t)n;
    const bool one_segment = hits || occluded;
    Q.t_min = one_segment ? t_min : 0.0f;            // ray_colour calls objs_hit with (0, 1e9) (ray.fut:130)
    Q.t_max = one_segment ? t_max : 1000000000.0f;
    Q.max_depth = one_segment ? 1 : max_depth;
    Q.occluded = occluded;
    Q.k = multi ? k : 0;
    Q.counts = multi ? counts : nullptr;
    CUDA_TRY(ctx, cudaMemsetAsync(L.work_cursor, 0, 2 * sizeof(int32_t), L.stream));
    CUDA_TRY(ctx, launch_warpqueue(P, Q, lc, L.stream, &ctx->launches));
    CUDA_TRY(ctx, cudaGetLastError());
  }
  // this query reads the scene's device memory until here on lane 0 (release_scene_block waits for it)
  if (!p->last_use[0]) CUDA_TRY(ctx, cudaEventCreateWithFlags(&p->last_use[0], cudaEventDisableTiming));
  CUDA_TRY(ctx, cudaEventRecord(p->last_use[0], L.stream));
  p->used[0] = true;
  CUDA_TRY(ctx, cudaEventRecord(ctx->ev_stop, L.stream));
  ctx->have_timing = true;
  return 0;
}

}  // namespace

extern "C" {

int ray_b200_trace_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev, int64_t n,
                        float t_min, float t_max, struct ray_b200_hit *hits_dev) {
  return trace(ctx, p, rays_dev, n, t_min, t_max, 1, hits_dev, nullptr, nullptr, nullptr, false, 0, nullptr, "trace_hits");
}

int ray_b200_trace_paths(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev, int64_t n,
                         int32_t max_depth, float *rgb_dev, int32_t *segments_dev) {
  return trace(ctx, p, rays_dev, n, 0.0f, 1000000000.0f, max_depth, nullptr, rgb_dev, segments_dev, nullptr, false, 0, nullptr,
               "trace_paths");
}

int ray_b200_trace_occluded(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev,
                            int64_t n, float t_min, float t_max, uint8_t *occluded_dev) {
  return trace(ctx, p, rays_dev, n, t_min, t_max, 1, nullptr, nullptr, nullptr, occluded_dev, false, 0, nullptr,
               "trace_occluded");
}

int ray_b200_trace_multi_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, const float *rays_dev,
                              int64_t n, float t_min, float t_max, int32_t k, struct ray_b200_hit *hits_dev, int32_t *counts_dev) {
  return trace(ctx, p, rays_dev, n, t_min, t_max, 1, hits_dev, nullptr, nullptr, nullptr, true, k, counts_dev, "trace_multi_hits");
}

int64_t ray_b200_hit_size(void) { return (int64_t)sizeof(struct ray_b200_hit); }

}  // extern "C"
