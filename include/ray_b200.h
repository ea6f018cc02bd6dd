/*
 * ray_b200.h — extensions next to the Futhark-compatible ABI of ray.h.
 *
 * The reference has no samples-per-pixel, no custom scenes, no float framebuffer and no multi-GPU
 * (ray.fut:150-154, 171-174, 246-247); BASELINE.json's configs need all four.  Because
 * futhark/main.c must stay unmodified, every extension is reachable two ways:
 *   - environment variables read by futhark_context_new (RAY_SPP, RAY_KERNEL, RAY_RANK, RAY_WORLD,
 *     RAY_DEVICE), so the unmodified driver can use them, and
 *   - the explicit C entry points below (plain pointers and sizes; device pointers are raw
 *     CUDA device addresses, e.g. torch.Tensor.data_ptr()).
 *
 * Multi-GPU.  Two ways: (a) one process per GPU (torchrun): ray_b200_context_set_shard + ray_b200_render_shard_into, an
 * NCCL gather by the host, ray_b200_detile — see raytracers_b200/distributed.py; (b) ONE process, several devices:
 * RAY_GPUS=N (or tuning parameter "gpus") makes the context drive devices d..d+N-1; futhark_entry_prepare_scene replicates
 * the scene, futhark_entry_render renders interleaved tiles on every device and pulls the shards to device d with peer
 * copies over NVLink.  This is the mode an unmodified futhark/main.c uses.  In mode (b) the raw-pointer entry points
 * (ray_b200_render_into, ray_b200_render_shard_into) keep addressing device d's shard only.
 *
 * spp semantics (SURVEY.md §8d): sample s of pixel (row j, column i) uses
 *   u = (f32(i) + ox_s) / f32(W),  v = (f32(H - j) + oy_s) / f32(H),
 *   ox_s = frac(f32(s) * 0.7548776662f), oy_s = frac(f32(s) * 0.5698402909f)   [ox_0 = oy_0 = 0]
 * colours are summed in sample order in f32, multiplied by 1/spp, then quantised as ray.fut:158-162.
 * At spp = 1 this is bit-identical to the reference's render.
 *
 * Quantisation: each channel is (int32)(255.99f * c) truncated toward 0, or INT32_MIN where 255.99f * c is NaN or
 * outside [-2^31, 2^31), and the pixel is (r << 16 | g << 8 | b) with 32-bit wrapping shifts.  That is what the
 * reference's multicore build computes on x86-64 (its C cast compiles to cvttss2si); a CUDA build of it would saturate
 * instead.  Colours outside [0, 1] (e.g. 0-255 colours), inf * 0 light and NaN camera rays (a camera looking along
 * vup or at its own position) reach it.  A NaN channel of the float framebuffer or of ray_b200_trace_paths is some
 * NaN: its bit pattern is not part of the contract.
 *
 * Ray queries ("ray queries" below): rays the caller made are traced against a prepared scene to their closest hit
 * (objs_hit), along their path (ray_colour), bit for bit, to their first accepted sphere (occlusion), or to the k
 * nearest of their accepted spheres (multi-hit), by the same warp-queue kernel in ray mode.  The last three also take
 * rays that carry their own (t_min, t_max) (struct ray_b200_ray, the *_ranged entry points).
 */
#ifndef RAY_B200_EXT_H
#define RAY_B200_EXT_H

#include "ray.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Render kernels (tuning param "kernel" / env RAY_KERNEL). */
enum ray_b200_kernel {
  RAY_B200_KERNEL_AUTO = 0,       /* the fastest measured variant (see resolve_kernel in api.cu) */
  RAY_B200_KERNEL_MEGA = 1,       /* one thread per pixel, whole ray_colour loop (parity anchor) */
  RAY_B200_KERNEL_PERSISTENT = 2, /* persistent CTAs, TMA-staged BVH, per-lane dynamic path refill */
  RAY_B200_KERNEL_WAVEFRONT = 3,  /* per-bounce persistent kernel + global ray queues + warp-vote compaction */
  RAY_B200_KERNEL_WARPQUEUE = 4,  /* persistent; lanes bound to (ray,node) items on warp-private smem queues */
  RAY_B200_KERNEL_STREAMQUEUE = 5,/* the same without rounds: per-ray item counters, finished rays refilled continuously */
  RAY_B200_KERNEL_LANEWALK = 6    /* persistent; a lane owns a ray's whole traversal (private smem stack), paths live in
                                     warp-shared slots, finished segments are shaded in dense batches, no rounds */
};

/* ---- context extensions ---------------------------------------------------------------------- */
/* Launch all work of this context on `cuda_stream` (a cudaStream_t / CUstream, e.g.
 * torch.cuda.Stream.cuda_stream).  NULL restores the context's own stream; pass cudaStreamLegacy
 * ((cudaStream_t)0x1) for the legacy default stream (whose raw handle is 0). */
int ray_b200_context_set_stream(struct futhark_context *ctx, void *cuda_stream);
/* Samples per pixel used by futhark_entry_render (default 1 = the reference). */
int ray_b200_context_set_spp(struct futhark_context *ctx, int32_t spp);
int ray_b200_context_set_kernel(struct futhark_context *ctx, int32_t kernel);
/* This process renders tiles t with t % world == rank (8x4-pixel tiles, row-major tile order). */
int ray_b200_context_set_shard(struct futhark_context *ctx, int32_t rank, int32_t world);
int ray_b200_context_device(struct futhark_context *ctx);
/* Device time in ms of the last render (CUDA events on the context's stream; syncs). */
int ray_b200_context_last_render_ms(struct futhark_context *ctx, float *ms);
/* Number of kernel launches issued by this context since creation. */
int64_t ray_b200_context_launch_count(struct futhark_context *ctx);
/* Diagnostic: while enabled, every warp of the warp-queue kernel records when it ran out of work.
 * ray_b200_context_warp_trace returns, for the last traced render, each warp's exit time in microseconds after
 * the first CTA started (exit_us may be NULL to query *count = SMs x warps per CTA).  Syncs the stream. */
int ray_b200_context_trace_warps(struct futhark_context *ctx, int32_t enable);
int ray_b200_context_warp_trace(struct futhark_context *ctx, float *exit_us, int64_t capacity, int64_t *count);

/* ---- scenes ------------------------------------------------------------------------------------ */
/* spheres: n x 7 floats (pos.xyz, colour.xyz, radius) — the `sphere` record of ray.fut:22-24;
 * cam7: look_from.xyz, look_at.xyz, fov — the rest of `scene`, ray.fut:171-174.  n >= 2 (bvh.fut:65). */
int ray_b200_scene_from_arrays(struct futhark_context *ctx, struct futhark_opaque_scene **out0,
                               const float *spheres, int64_t n, const float *cam7);
/* SURVEY.md §8d config 5: splitmix64(seed) stream, 7 draws per sphere, camera (0,0,1100)->(0,0,0). */
int ray_b200_scene_random(struct futhark_context *ctx, struct futhark_opaque_scene **out0, int64_t n,
                          uint64_t seed);
int64_t ray_b200_scene_num_spheres(struct futhark_context *ctx, const struct futhark_opaque_scene *s);
int ray_b200_scene_get_arrays(struct futhark_context *ctx, const struct futhark_opaque_scene *s, float *spheres,
                              float *cam7);

/* ---- prepared scene introspection (tests compare these with the oracle's LBVH) ----------------- */
struct ray_b200_bvh_info {
  int64_t n_leaves, n_inner;
  int32_t max_depth, refit_sweeps, stale_nodes, smem_nodes;
  float root_box[6];
  float camera[12]; /* origin, llc, horizontal, vertical (ray.fut:88-91) */
};
int ray_b200_prepared_info(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           struct ray_b200_bvh_info *info);
/* Karras-order dump: morton[n], perm[n], left/right/parent[n-1] (leaf i = ~i), boxes[(n-1)*6]. NULLs skipped. */
int ray_b200_prepared_dump(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           uint32_t *morton, int32_t *perm, int32_t *left, int32_t *right, int32_t *parent,
                           float *boxes);

/* The packed BVH2C arrays as they sit in HBM (tests compare device-built and host-built scenes):
 * nodes / nodes_soa: (n-1) x 16 floats, geom / colour: n x 4 floats.  NULLs skipped.  Synchronous. */
int ray_b200_prepared_packed(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, float *nodes,
                             float *nodes_soa, float *geom, float *colour);
/* Bytes prepare_scene copies host -> device: the sphere records (LBVH build and packing run on the device);
 * with tuning "host_build" / RAY_HOST_BUILD=1 the host-built arrays instead. */
int64_t ray_b200_prepared_upload_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p);
/* Bytes of the prepared scene resident in HBM (packed BVH2C + the Karras-order LBVH kept for introspection). */
int64_t ray_b200_prepared_device_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p);
/* Runs prepare_scene's device work again for an existing handle: H2D of the sphere records from page-locked
 * memory + LBVH build on the device (the H2D leg of bench.py's end-to-end step). */
int ray_b200_prepared_reupload(struct futhark_context *ctx, struct futhark_opaque_prepared_scene *p);

/* ---- render extensions -------------------------------------------------------------------------- */
/* render with explicit spp; optional float framebuffer.  out_pix_dev: device int32[h][w] (REQUIRED);
 * out_rgb_dev: device float[h][w][3] (or NULL).  Asynchronous on the context's stream.
 * With a shard set (world > 1) only this rank's pixels are written.  On a single-process multi-GPU context
 * (RAY_GPUS > 1) this call, ray_b200_render_shard_into and ray_b200_render_batch return an error: only
 * futhark_entry_render / ray_b200_entry_render_spp gather the helper devices' tiles. */
int ray_b200_render_into(struct futhark_context *ctx, int32_t *out_pix_dev, float *out_rgb_dev, int64_t h,
                         int64_t w, int32_t spp, const struct futhark_opaque_prepared_scene *p);
/* Same, host buffers: H2D of nothing (the scene is resident), D2H of the frame, synchronous.
 * This is the call bench.py's e2e leg times. */
int ray_b200_render_host(struct futhark_context *ctx, int32_t *out_pix_host, float *out_rgb_host, int64_t h,
                         int64_t w, int32_t spp, const struct futhark_opaque_prepared_scene *p);
/* Progressive rendering: samples [s_begin, s_end) of every pixel of an h x w frame, added to a running sum, so that a
 * caller can show a preview after a few samples and refine it without re-tracing anything.
 * accum_dev: device float[h][w][3], row-major.  On entry, when s_begin > 0, it holds each pixel's running sum (for
 * example from earlier calls); it is not read when s_begin == 0.  On return it holds sum + colour_{s_begin} + ... +
 * colour_{s_end-1}, added one sample at a time in sample order in f32.  When s_begin == 0 the sum starts as colour_0
 * itself, not 0 + colour_0 (this keeps -0.0).  out_pix_dev / out_rgb_dev (each may be NULL): the frame at spp = s_end,
 * exactly what ray_b200_render_into(spp = s_end) writes.
 *   Exactness: any chain of calls [0, a), [a, b), ..., [y, S) on one buffer leaves the same accum as one call [0, S), bit
 *   for bit, and its pixels and float framebuffer equal ray_b200_render_into(spp = S) (NaN-aware: a NaN is some NaN).
 *   The sum read at s_begin > 0 is whatever the caller left in the buffer; the result is the f32 arithmetic above on it.
 *   Sample s is sample s of the spp semantics above, whatever the chunking.
 *   The call is asynchronous on the context's stream; stream order, the pipeline lanes, freeing the prepared scene while
 *   the call is in flight, ray_b200_context_last_render_ms and ray_b200_context_launch_count (one launch per call) behave
 *   as for ray_b200_render_into.  With a shard set (world > 1) only this rank's pixels of accum and of the outputs are
 *   read or written, in the row-major layout; there is no tile-major form.
 *   It runs on the warp-queue kernel whatever RAY_KERNEL or the context's kernel says (every kernel's frames are
 *   bit-identical).
 *   Errors (nonzero return, futhark_context_get_error; the context stays usable): every error of ray_b200_render_into
 *   (an s_end it would reject as spp, a RAY_GPUS > 1 context, ...), s_begin < 0, s_end <= s_begin, accum_dev == NULL. */
int ray_b200_render_accumulate(struct futhark_context *ctx, float *accum_dev, int64_t h, int64_t w,
                               int32_t s_begin, int32_t s_end, int32_t *out_pix_dev, float *out_rgb_dev,
                               const struct futhark_opaque_prepared_scene *p);
/* Several views of one prepared scene in one launch, each with its own camera, sharing the scene's BVH: a camera
 * fly-through over a static scene, a stereo pair, the six faces of a cube map, a batch of poses, or (n_views = 1) the
 * prepared scene seen from another camera without preparing it again.
 * cams7_host: host float[n_views][7] = look_from.xyz, look_at.xyz, fov of each view (the cam7 layout of
 * ray_b200_scene_from_arrays).  out_pix_dev: device int32[n_views][h][w] (required); out_rgb_dev: device
 * float[n_views][h][w][3] or NULL.
 *   Exactness: view v's pixels and float framebuffer are bit for bit what ray_b200_render_into(h, w, spp) writes for
 *   prepare_scene(h, w, S_v), where S_v is the prepared scene's spheres with cams7[v] as its camera.  That camera is
 *   make_camera of cams7[v] with the aspect ratio f32(w) / f32(h) of this call (ray.fut:243-244), computed on the host
 *   as prepare_scene computes it (ray_b200_host_camera gives the same 12 floats).  The spp semantics and the
 *   quantisation rule above hold unchanged.  A NaN camera (a view looking along vup or at its own position) quantises by
 *   that rule and does not affect the other views; a NaN of the float framebuffer is some NaN.
 *   The call is asynchronous on the context's stream and is one kernel launch (plus the heavy-first probe when enabled
 *   and spp > 1, as for ray_b200_render_into).  cams7_host may be reused once the call returns: the library copies the
 *   camera table to stream-ordered device memory and frees it behind the launch.  ray_b200_context_last_render_ms,
 *   ray_b200_context_launch_count, the pipeline lanes, and freeing or re-uploading the prepared scene while the call is
 *   in flight behave as for ray_b200_render_into.
 *   It runs on the warp-queue kernel whatever RAY_KERNEL or the context's kernel says, and leaves the prepared scene's
 *   learned claim order untouched: renders before and after it plan and launch exactly as without it.
 *   Errors (nonzero return, futhark_context_get_error; the context stays usable): every error of ray_b200_render_into
 *   (image size, spp, an invalid prepared scene, a RAY_GPUS > 1 context), n_views < 1, cams7_host == NULL,
 *   out_pix_dev == NULL, n_views x tiles(h, w) > 2^25 (at most 2^30 padded pixels over all views, where a tile is 8 x 4
 *   pixels), and a shard set (world > 1). */
int ray_b200_render_views_into(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                               const float *cams7_host, int32_t n_views, int64_t h, int64_t w, int32_t spp,
                               int32_t *out_pix_dev, float *out_rgb_dev);
/* Like futhark_entry_render but with explicit spp (library-owned result). */
int ray_b200_entry_render_spp(struct futhark_context *ctx, struct futhark_i32_2d **out0, int64_t h, int64_t w,
                              int32_t spp, const struct futhark_opaque_prepared_scene *p);

/* ---- ray queries: caller-supplied rays against a prepared scene ----------------------------------------
 * The two queries of the reference, for any ray: the closest hit of objs_hit (ray.fut:76-86) and the colour of
 * ray_colour (ray.fut:126-148), bit for bit, on the warp-queue kernel in ray mode (whatever RAY_KERNEL / the context's
 * kernel says; a shard setting is ignored: rays are not tiles).  On a RAY_GPUS > 1 context they run on device d, which
 * holds the scene.  rays_dev: device float[n][6] = origin.xyz, dir.xyz (dir need not be normalised; zero components and
 * an all-zero direction are fine; rays with non-finite components are outside the contract).  Asynchronous on the
 * context's stream; ray_b200_context_last_render_ms and ray_b200_context_launch_count count them like renders, and a
 * prepared scene may be freed or re-uploaded while a query that reads it is in flight.
 * Errors (nonzero return, futhark_context_get_error; the context stays usable): n < 0 or n > 2^30, a NULL required
 * pointer with n > 0, an invalid prepared scene, t_min < 0, a non-finite t_min or t_max, max_depth outside [0, 65535].
 * n == 0 does nothing.  t_max <= t_min is legal: every ray misses. */
/* Closest hit of ray i = objs_hit objs r t_min t_max (ray.fut:76-86), bit for bit. */
struct ray_b200_hit {
  float t;          /* -1 when there is no hit (a hit always has t > t_min >= 0) */
  int32_t sphere;   /* index into the scene's sphere array as given (scene_from_arrays / scene_get_arrays order), -1 = none */
  float p[3];       /* point_at_param r t (ray.fut:14-15); 0 when there is no hit */
  float normal[3];  /* scale (1/radius) (p - centre) (ray.fut:42-43); 0 when there is no hit */
};                  /* 32 bytes */
/* Boxes are tested against (t_min, t_max), spheres with epsilon 0.1 whatever t_min is (ray.fut:77-79), the winner is
 * re-intersected with (t_min, t_best + 1) (ray.fut:85; a failed re-intersection is no hit), and on equal t the lowest
 * Morton-sorted leaf wins.  hits_dev: device struct ray_b200_hit[n]. */
int ray_b200_trace_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                        const float *rays_dev, int64_t n, float t_min, float t_max, struct ray_b200_hit *hits_dev);
/* Colour of ray i = ray_colour objs r max_depth (ray.fut:126-148), bit for bit, before quantisation; every segment
 * uses (0, 1e9) as ray_colour does.  rgb_dev: device float[n][3]; segments_dev: device int32[n] = objs_hit calls of
 * the path (or NULL).  Camera rays of a frame through this call, quantised, equal the frame. */
int ray_b200_trace_paths(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                         const float *rays_dev, int64_t n, int32_t max_depth, float *rgb_dev, int32_t *segments_dev);
/* Occlusion (shadow / visibility rays): occluded_dev[i] = 1 if the reference's bvh_fold (bvh.fut:61-84) reaches some leaf
 * whose sphere_hit L[i] r t_min t_max (ray.fut:32-51) is a hit, boxes tested against (t_min, t_max) as objs_hit tests
 * them, else 0.  Unlike ray_b200_trace_hits there is no epsilon 0.1 (t_min bounds the sphere tests too) and no
 * re-intersection, and the occluding sphere is not reported.  The answer is an OR over the reached leaves, so it does
 * not depend on traversal order, and a ray's traversal stops at its first accepted sphere.  At t_min = 0.1 it equals
 * "ray_b200_trace_hits(t_min = 0.1, t_max) reports a hit" for every ray whose closest hit has t < 2^24.
 * occluded_dev: device uint8_t[n] (a torch.bool buffer).  Point-to-point visibility: origin = the point, direction =
 * target - origin (not normalised), and an interval such as (1e-4, 1 - 1e-4), which excludes both end points. */
int ray_b200_trace_occluded(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                            const float *rays_dev, int64_t n, float t_min, float t_max, uint8_t *occluded_dev);
/* Multi-hit (transparency layers, depth complexity, line-of-sight lists): A(r) = the leaves the reference's bvh_fold
 * (bvh.fut:61-84) reaches, boxes tested against (t_min, t_max) as objs_hit tests them, whose sphere_hit L[i] r t_min
 * t_max (ray.fut:32-51) is a hit, each with its t (root1 if it lies in the interval, else root2).  As in
 * ray_b200_trace_occluded there is no epsilon 0.1 and no re-intersection, and a sphere gives at most one record, its
 * first intersection in the interval.  A(r) is ordered by ascending t, then ascending Morton-sorted leaf (coincident
 * identical spheres: ascending caller index).  hits_dev[i][j], j < min(k, |A(r)|): the j-th member as struct
 * ray_b200_hit, t, sphere, p and normal made as ray_b200_trace_hits makes them; the remaining records are t = -1,
 * sphere = -1, p = normal = 0.  counts_dev[i] = |A(r)|, not capped at k.  The set of reached leaves does not depend
 * on traversal order, so neither do the records nor the count.  Two identities hold exactly:
 *   counts_dev[i] > 0  ==  ray_b200_trace_occluded(t_min, t_max) for every ray;
 *   at t_min = 0.1, record 0 == the ray_b200_trace_hits(0.1, t_max) record, all 8 words, for every ray whose closest
 *   hit has t < 2^24.
 * hits_dev: device struct ray_b200_hit[n][k] (record offsets are 64-bit: n * k may pass 2^32); counts_dev: device
 * int32[n] or NULL.  Further errors: k outside [1, 64]. */
int ray_b200_trace_multi_hits(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                              const float *rays_dev, int64_t n, float t_min, float t_max, int32_t k,
                              struct ray_b200_hit *hits_dev, int32_t *counts_dev);
/* sizeof(struct ray_b200_hit) as the library was compiled (32). */
int64_t ray_b200_hit_size(void);
/* Ranged queries: rays that carry their own interval, as Embree's tnear / tfar, OptiX's tmin / tmax and DXR's RayDesc do
 * (shadow rays to many lights with unit directions and t_max = each light's distance, per-ray near / far clipping, the
 * closest hit over two prepared scenes by tracing the second with t_max = the first one's t).  rays_dev: device
 * struct ray_b200_ray[n], 4-byte aligned (a 16-byte aligned buffer is read with 16-byte loads).
 * The answer for ray i is exactly what the per-call entry point returns for that ray alone, called with
 * (rays[i].t_min, rays[i].t_max).
 * A ray whose t_min is not finite and >= 0 (-0.0 is valid), or whose t_max is not finite, is not an error (the host does
 * not read the rays): it gets the empty answer that t_max <= t_min gives, t = -1 / sphere = -1 / p = normal = 0,
 * occluded = 0, k empty records and a count of 0, and the other rays are unaffected.  Errors are those of the per-call
 * entry points without the interval checks: n outside [0, 2^30], a NULL buffer with n > 0, an invalid prepared scene,
 * k outside [1, 64].  There is no ranged trace_paths: ray_colour uses (0, 1e9) for every segment.
 * Continuing a multi-hit list past k from the last record's t is not exact: a sphere that straddles the new t_min gives
 * its second root, records at exactly that t are dropped (the interval is open), and the stale boxes of the fixed-sweep
 * refit make the set of reached leaves depend on the interval. */
struct ray_b200_ray {
  float o[3];   float t_min;   /* origin, near end of the interval */
  float d[3];   float t_max;   /* direction (need not be normalised), far end */
};              /* 32 bytes */
int ray_b200_trace_hits_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                               const struct ray_b200_ray *rays_dev, int64_t n, struct ray_b200_hit *hits_dev);
int ray_b200_trace_occluded_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                                   const struct ray_b200_ray *rays_dev, int64_t n, uint8_t *occluded_dev);
int ray_b200_trace_multi_hits_ranged(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                                     const struct ray_b200_ray *rays_dev, int64_t n, int32_t k,
                                     struct ray_b200_hit *hits_dev, int32_t *counts_dev);
/* sizeof(struct ray_b200_ray) as the library was compiled (32). */
int64_t ray_b200_ray_size(void);

/* ---- multi-GPU tile sharding (one process per GPU; the gather itself is NCCL, done by the host) -- */
/* Number of 8x4 tiles rank `rank` of `world` owns for an h x w image, and the padded per-rank count
 * (equal on all ranks, so a plain all_gather / gather works). */
int64_t ray_b200_shard_tiles(int64_t h, int64_t w, int32_t rank, int32_t world);
int64_t ray_b200_shard_tiles_padded(int64_t h, int64_t w, int32_t world);
/* Renders this rank's tiles into a compact tile-major device buffer int32[tiles_padded][32]. */
int ray_b200_render_shard_into(struct futhark_context *ctx, int32_t *out_tiles_dev, int64_t h, int64_t w,
                               int32_t spp, const struct futhark_opaque_prepared_scene *p);
/* Several frames in one call, up to two of them in flight on the device, so that the long-path tail of one frame
 * is covered by the start of the next (the frames are independent: different prepared scenes, sizes or outputs).
 * For the caller the batch is ONE operation on the context's stream: it starts after earlier work on that stream, and
 * later work on that stream starts after every job has finished.  Jobs are launched in array order (put the frame
 * with the longest tail first).  ray_b200_context_last_render_ms then reports the whole batch. */
struct ray_b200_render_job {
  const struct futhark_opaque_prepared_scene *prepared;
  int64_t h, w;
  int32_t spp;          /* 0 = the context's default */
  int32_t shard_layout; /* 0: out_dev = int32[h][w], row-major (ray_b200_render_into);
                           1: out_dev = this rank's compact tiles int32[tiles_padded][32] (ray_b200_render_shard_into) */
  int32_t *out_dev;     /* device (may be a PEER device's memory mapped with ray_b200_ipc_open: row-major layout + a
                           shard set = every rank writes its own pixels straight into rank 0's frame over NVLink) */
  float *out_rgb_dev;   /* device float[h][w][3] or NULL (row-major layout only) */
  /* peer-frame protocol (all optional, NULL = off), see "peer-memory frames" below:
   * before the frame's kernel starts, its stream waits until *wait_flag >= wait_value (back-pressure from the consumer);
   * when the last warp of the frame's kernel has written its pixels, *done_flag is incremented by 1 (system scope). */
  uint32_t *wait_flag;
  uint32_t wait_value;
  uint32_t reserved0;
  uint32_t *done_flag;
};
int ray_b200_render_batch(struct futhark_context *ctx, const struct ray_b200_render_job *jobs, int32_t n);
/* Pipelined submission (off by default).  With it on, ray_b200_render_batch does NOT join its second lane back into the
 * context's stream: consecutive frames alternate between the two lanes ACROSS calls, each lane ordered only after its own
 * previous frame (and after earlier work on the context's stream, e.g. a scene re-upload), so frame k+1 starts on every
 * SM whose CTA of frame k has retired - a frame's last 50-bounce paths no longer idle the GPU at the end of every
 * batch.  The caller orders its reads itself (done_flag / ray_b200_flag_wait, or ray_b200_pipeline_join, or
 * futhark_context_sync, which waits for both lanes).  Prepared scenes may be freed or re-uploaded while frames that use
 * them are in flight: their device memory is reclaimed only after the last such frame (stream-ordered, on a third stream). */
int ray_b200_context_set_pipeline(struct futhark_context *ctx, int32_t on);
/* Makes the context's stream wait for every frame enqueued so far on either lane (no host synchronisation). */
int ray_b200_pipeline_join(struct futhark_context *ctx);
/* sizeof(struct ray_b200_render_job) as the library was compiled: lets a foreign-language binding check its layout. */
int64_t ray_b200_render_job_size(void);
/* gathered_dev: int32[world][tiles_padded][32] (rank-major, as produced by an NCCL gather);
 * writes the row-major image int32[h][w] to out_pix_dev. */
int ray_b200_detile(struct futhark_context *ctx, const int32_t *gathered_dev, int32_t *out_pix_dev, int64_t h,
                    int64_t w, int32_t world);

/* ---- peer-memory frames: the gather fused into the render kernel ----------------------------------------
 * One process per GPU.  Rank 0 allocates a ring of frames with ray_b200_ipc_alloc and hands the 64-byte handle to the
 * other ranks (any transport: torch.distributed object broadcast in raytracers_b200/distributed.py); they map it with
 * ray_b200_ipc_open and pass the mapped address as `out_dev` of a row-major render with their shard set.  The render
 * kernel's pixel stores then ARE the collective: they travel over NVLink into rank 0's frame, no tile buffer, no
 * ncclGather, no de-tiling kernel.  Completion and back-pressure are two 32-bit flags per frame slot in the same
 * allocation (done_flag / wait_flag of ray_b200_render_job); the consumer side enqueues ray_b200_flag_wait on its copy
 * stream, copies the frame out and publishes the slot again with ray_b200_flag_set. */
#define RAY_B200_IPC_HANDLE_BYTES 64
int ray_b200_ipc_alloc(struct futhark_context *ctx, int64_t bytes, void **dev_ptr, unsigned char *handle64);
int ray_b200_ipc_free(struct futhark_context *ctx, void *dev_ptr);
int ray_b200_ipc_open(struct futhark_context *ctx, const unsigned char *handle64, void **dev_ptr);
int ray_b200_ipc_close(struct futhark_context *ctx, void *dev_ptr);
/* Enqueue on `stream` (a cudaStream_t; NULL = the context's stream): spin until *flag >= value (system-scope acquire;
 * gives up after timeout_ms and records an error that the next ray_b200_flag_status call returns). */
int ray_b200_flag_wait(struct futhark_context *ctx, void *stream, uint32_t *flag_dev, uint32_t value, int32_t timeout_ms);
/* Enqueue on `stream`: *flag = value (system-scope release). */
int ray_b200_flag_set(struct futhark_context *ctx, void *stream, uint32_t *flag_dev, uint32_t value);
/* Number of flag waits that timed out since the context was created (0 = healthy). */
int ray_b200_flag_status(struct futhark_context *ctx, int64_t *timeouts);
/* Enqueue on `stream`: device -> host copy (host_dst should be page-locked for the copy to be asynchronous). */
int ray_b200_copy_to_host_async(struct futhark_context *ctx, void *stream, void *host_dst, const void *dev_src, int64_t bytes);

/* ---- work counters (roofline numerators) ---------------------------------------------------------- */
struct ray_b200_counters { uint64_t segments, node_steps, box_tests, leaf_tests; };
/* Re-renders (1 spp) with counting kernels and returns the work the GPU traversal did. */
int ray_b200_count_work(struct futhark_context *ctx, int64_t h, int64_t w, int32_t spp,
                        const struct futhark_opaque_prepared_scene *p, struct ray_b200_counters *out);

/* ---- host-only entry points (no context, no device needed): the setup path's host logic ------------ */
/* name: "rgbbox" | "irreg" | "random" (n, seed used by "random" only).  spheres may be NULL to query *count. */
int ray_b200_host_scene(const char *name, int64_t n, uint64_t seed, float *spheres, int64_t capacity, float *cam7,
                        int64_t *count);
/* camera look_from look_at (0,1,0) fov (w/h)  (ray.fut:93-107, 243-244) -> origin, llc, horizontal, vertical */
int ray_b200_host_camera(const float *cam7, int64_t h, int64_t w, float *out12);
/* bvh_mk (bvh.fut:30-59) in Karras order; info4 = {refit_sweeps, max_depth, stale_nodes, 0}. 2 = n < 2. */
int ray_b200_host_lbvh(const float *spheres, int64_t n, uint32_t *morton, int32_t *perm, int32_t *left,
                       int32_t *right, int32_t *parent, float *boxes, int32_t *info4);
void ray_b200_host_sample_offsets(int32_t spp, float *table);

const char *ray_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* RAY_B200_EXT_H */
