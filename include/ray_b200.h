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
  RAY_B200_KERNEL_AUTO = 0,       /* the fastest measured variant (see resolve_kernel in api_render.cu) */
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
/* What a launch traces (struct ray_b200_plan's query): a frame, a chunk of a progressive frame, several views, the
 * selected pixels of an adaptive progressive frame (ADAPTIVE_VAR: with their sample variance), the first hits of a frame's
 * camera rays (GBUFFER: ray_b200_render_gbuffer), one frame of each scene of a scene batch (SCENE_BATCH:
 * ray_b200_render_scene_batch_into), or the caller's rays to their closest hit or along their path (trace_hits /
 * trace_paths), to their first hit (occlusion), or to their k nearest hits (multi-hit), and the same three kinds of ray
 * query on the scenes of a scene batch (SCENE_BATCH_CLOSEST for hits and paths, SCENE_BATCH_ANYHIT, SCENE_BATCH_MULTIHIT:
 * ray_b200_scene_batch_trace_*). */
enum ray_b200_query {
  RAY_B200_QUERY_PIXELS = 0, RAY_B200_QUERY_CLOSEST = 1, RAY_B200_QUERY_ANYHIT = 2, RAY_B200_QUERY_MULTIHIT = 3,
  RAY_B200_QUERY_ACCUMULATE = 4, RAY_B200_QUERY_VIEWS = 5, RAY_B200_QUERY_ADAPTIVE = 6, RAY_B200_QUERY_ADAPTIVE_VAR = 7,
  RAY_B200_QUERY_GBUFFER = 8, RAY_B200_QUERY_SCENE_BATCH = 9, RAY_B200_QUERY_SCENE_BATCH_CLOSEST = 10,
  RAY_B200_QUERY_SCENE_BATCH_ANYHIT = 11, RAY_B200_QUERY_SCENE_BATCH_MULTIHIT = 12
};
/* The plan of the last render kernel launch on the context: the last frame, progressive chunk, views call or ray query
 * (for ray_b200_render_batch, its last job), as it was launched.  Calls that launch no render kernel (a query of n = 0
 * rays or of max_depth 0, ray_b200_count_work, the helper devices of a RAY_GPUS > 1 context) leave it unchanged; before
 * the first launch it is all zeros (kernel 0).  For a kernel other than the warp-queue kernel only kernel, query and the
 * staging fields are set.  It shows which of the warp-queue kernel's instantiations ran: the test-suite checks that
 * every one of them is reached and exact.  Host-only, does not synchronise. */
struct ray_b200_plan {
  int32_t kernel;        /* enum ray_b200_kernel of the launched kernel; 0 = nothing launched yet */
  int32_t query;         /* enum ray_b200_query */
  int32_t ranged;        /* 1: the rays carried their own intervals (the *_ranged queries) */
  int32_t k;             /* rays in flight per warp / 32 (1 or 2) */
  int32_t warps, ctas;   /* warps per CTA, CTAs launched (at most one per SM) */
  int32_t spread;        /* 1: the samples of a pixel were spread over a warp's slots (a finished-sample buffer was used) */
  int32_t packet;        /* packet-walk threshold (lanes per node step); 0 = no packet walk */
  int32_t all_nodes;     /* 1: every BVH node was staged in shared memory */
  int32_t spheres;       /* 1: every sphere record was staged as well */
  int32_t ncap, nlow;    /* node-queue allocation (entries); breadth-first node batches below nlow queued items */
  int32_t smem_nodes;    /* BVH nodes staged in shared memory (a BFS prefix) */
  int32_t smem_spheres;  /* sphere records staged (0 or n_leaves) */
  int32_t n_inner, n_leaves;
  int64_t stage_budget;  /* shared memory (bytes) the kernel's queues left for staging, before the stage_cap tuning cap */
  int64_t dynamic_smem;  /* dynamic shared memory requested per CTA (bytes) */
};
int ray_b200_context_last_plan(struct futhark_context *ctx, struct ray_b200_plan *out);
/* sizeof(struct ray_b200_plan) as the library was compiled (80). */
int64_t ray_b200_plan_size(void);

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
 * with tuning "host_build" / RAY_HOST_BUILD=1 the host-built arrays instead.  0 for a scene last built by
 * ray_b200_prepare_scene_device or ray_b200_prepared_update (and re-uploaded since), except on a host_build context. */
int64_t ray_b200_prepared_upload_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p);
/* Bytes of the prepared scene resident in HBM (packed BVH2C + the Karras-order LBVH kept for introspection). */
int64_t ray_b200_prepared_device_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p);
/* Runs prepare_scene's device work again for an existing handle: H2D of the sphere records from page-locked
 * memory + LBVH build on the device (the H2D leg of bench.py's end-to-end step).  For a scene last built from device
 * memory (below) the records are recovered on the device from the scene's own arrays instead, with no H2D copy. */
int ray_b200_prepared_reupload(struct futhark_context *ctx, struct futhark_opaque_prepared_scene *p);

/* ---- prepared scenes from device memory: dynamic scenes without a host round trip -------------------------------
 * A caller whose spheres live in device memory (a simulation, a learned model, an animation computed on the GPU) builds
 * and rebuilds a prepared scene from them directly.  spheres_dev: device float[n][7] in the layout of
 * ray_b200_scene_from_arrays (pos.xyz, colour.xyz, radius), 4-byte aligned, readable by the context's device;
 * cam7_host: host float[7] as there.
 *   Exactness.  After ray_b200_prepare_scene_device(h, w, S, n, cam7) or ray_b200_prepared_update(p, S, n, cam7) the
 *   prepared scene is bit for bit the one futhark_entry_prepare_scene(h, w, scene_from_arrays(S, n, cam7)) makes from
 *   the same 7n floats (on update with cam7_host == NULL, cam7 is the scene's own camera): prepared_info (refit_sweeps,
 *   stale_nodes, max_depth and the root box included), prepared_dump, prepared_packed, every frame and every ray query.
 *   The build is prepare_scene's LBVH build, only fed from device memory.  There is no refit-only update: a refit that
 *   kept the old topology would give a tree other than the reference's, whose stale boxes decide which hits are culled,
 *   so its frames would not be the reference's.
 *   No host copy.  The calls copy no records host -> device (ray_b200_prepared_upload_bytes is 0), and the library
 *   keeps no host copy of them.  Where it needs them it recovers them on the device from the packed arrays,
 *   sphere[perm[k]] = (geom[k].xyz, colour[k].xyz, geom[k].w), which is exact: ray_b200_prepared_spheres (one gather
 *   launch), futhark_store_opaque_prepared_scene (which then reads them back and synchronises) and
 *   ray_b200_prepared_reupload (which rebuilds from the recovered records on the device).
 *   Stream order and blocking.  spheres_dev is read on the context's stream, after the work enqueued there before the
 *   call; a producer on another stream must be ordered before it (ray_b200_context_set_stream, or an event).  Like
 *   prepare_scene, both calls return after the build's 32-byte read-back, because render planning needs the tree
 *   depth; spheres_dev may then be reused or freed.  (A non-blocking update would need planning without the depth; it
 *   is not offered.)
 *   Frames in flight.  Frames, queries and batches enqueued before an update read the old tree, whose memory is freed
 *   behind them on either pipeline lane; work enqueued after it reads the new tree.  The new tree is built before the old
 *   one is released, so an update whose build fails leaves the previous tree in place.
 *   Learned claim order.  An update drops the scene's learned claim order: the renders after it plan and launch as the
 *   first renders of a freshly prepared scene do.
 *   Context state.  ray_b200_context_last_plan and last_render_ms are unchanged; ray_b200_context_launch_count counts
 *   the build's launches as for prepare_scene.
 *   host_build contexts (RAY_HOST_BUILD=1): the records are read back and the host builder runs; the result is the
 *   same, and ray_b200_prepared_upload_bytes is the block's, as for prepare_scene there.
 *   Errors (nonzero return and a message; the context stays usable, and an argument error leaves an existing prepared
 *   scene unchanged and usable): n < 2 or n > 2^26, a NULL spheres_dev, out0, p or (for prepare_scene_device)
 *   cam7_host, spheres_dev not readable by the device (plain host memory), h <= 0 or w <= 0, an invalid prepared scene,
 *   and a RAY_GPUS > 1 context (its helper devices would need the records). */
int ray_b200_prepare_scene_device(struct futhark_context *ctx, struct futhark_opaque_prepared_scene **out0, int64_t h,
                                  int64_t w, const float *spheres_dev, int64_t n, const float *cam7_host);
/* Replaces the spheres of an existing prepared scene (any n in [2, 2^26]) and rebuilds its tree in place, for its
 * (h, w); cam7_host == NULL keeps the camera, otherwise the camera is remade from cam7_host for the scene's (h, w). */
int ray_b200_prepared_update(struct futhark_context *ctx, struct futhark_opaque_prepared_scene *p,
                             const float *spheres_dev, int64_t n, const float *cam7_host);
/* The prepared scene's current sphere records, in the caller's order, bit for bit as given (by any of the calls that
 * make or update a prepared scene): spheres_dev = device float[n][7] (NULL: not written; n = prepared_info's n_leaves),
 * written by one gather launch, asynchronous on the context's stream; cam7_host = host float[7] (NULL: not written).
 * Errors: an invalid prepared scene. */
int ray_b200_prepared_spheres(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                              float *spheres_dev, float *cam7_host);

/* ---- scene batches: many small scenes, built and rendered together ------------------------------------------------
 * A caller with B scenes in device memory (vectorised environments, a dataset generator, a sweep over a model's
 * outputs) builds all B trees in one pass and renders one frame of every scene in one launch, instead of one prepare and
 * one render call per scene.  spheres_dev: device float[B][n][7], scene b's records at b n 7, each scene in the layout
 * of ray_b200_scene_from_arrays, 4-byte aligned, readable by the context's device; cams7_host: host float[B][7], scene
 * b's camera as there.  B = n_scenes >= 1, 2 <= n, B n <= 2^26.
 *   Ragged batches.  ray_b200_scene_batch_new_ragged builds B scenes of different sizes: scene b has counts_host[b] =
 *   n_b >= 2 spheres (host int64[B], N = n_0 + .. + n_{B-1} <= 2^26), packed back to back in spheres_dev = device
 *   float[N][7], scene b's records from row off_b = n_0 + .. + n_{b-1}.  Everything below holds for it with S + 7 n b
 *   read as S + 7 off_b and n as n_b: member b is bit for bit ray_b200_prepare_scene_device(h, w, S + 7 off_b, n_b,
 *   cams7 + 7 b), including its refit_sweeps, trunc(log2f(n_b)) + 2, and the stale boxes that count leaves (no padding
 *   sphere could keep them: it would move the box the Morton keys are quantised in).  A uniform batch is a ragged batch
 *   whose counts are equal: new_device(B, n) and new_ragged with B counts n make the same batch, bit for bit.
 *   ray_b200_scene_batch_update_ragged rebuilds every member from new records and new counts (B stays; counts may
 *   differ from the current ones), as update does; ray_b200_scene_batch_update on a batch whose counts differ is an
 *   error that changes nothing.  ray_b200_scene_batch_shape reports n = the common count, or 0 when the members differ;
 *   ray_b200_scene_batch_counts writes the B counts to counts_host (host int64[B]).  Frames and every
 *   ray_b200_scene_batch_trace_* take a ragged batch as they are; the sphere of a hit record indexes scene b's own
 *   records, in [0, n_b).  Errors, on top of new_device's: a NULL counts_host, a count < 2, N > 2^26, and spheres_dev
 *   not device-readable.
 *   Exactness.  Member b of ray_b200_scene_batch_new_device(h, w, S, B, n, cams7) is bit for bit the prepared scene
 *   ray_b200_prepare_scene_device(h, w, S + 7 n b, n, cams7 + 7 b) makes: ray_b200_scene_batch_member returns it, and its
 *   prepared_info (every field), prepared_dump, prepared_packed, prepared_spheres, frames and ray queries are that
 *   scene's.  Frame b of ray_b200_render_scene_batch_into(h, w, spp) is ray_b200_render_into(h, w, spp) of member b, bit
 *   for bit (pixels, and the float framebuffer including its NaNs).
 *   One build, one read-back.  The build runs the kernels of prepare_scene's device build once over all B scenes (a
 *   stable sort of (scene, Morton key) is each scene's own sort) and ends in one read-back of B x 32 bytes, the members'
 *   depths, stale counts and root boxes: one synchronisation per batch.  The cameras are made on the host for the
 *   build's (h, w) as prepare_scene makes them (the aspect ratio w / h), and kept on the device with the root boxes.
 *   One launch.  ray_b200_render_scene_batch_into renders frame b of scene b for every b in one launch of the warp-queue
 *   kernel (the h, w of the call set the pixel grid; the cameras are those of the build's h, w, as for a prepared
 *   scene), planned over all B trees together.  ray_b200_context_last_plan reports RAY_B200_QUERY_SCENE_BATCH;
 *   last_render_ms and launch_count count it as a render.  The tiles are claimed in the plain chunk permutation (no
 *   heavy-first probe, no learned claim order), and no prepared scene's learned order is touched.
 *   Outputs.  out_pix_dev: device int32[B][h][w] (required), frame b at b h w; out_rgb_dev: device float[B][h][w][3] or
 *   NULL.  Asynchronous on the context's stream.
 *   Update.  ray_b200_scene_batch_update rebuilds every member from new records of the same B and n (and new cameras,
 *   or cams7_host == NULL to keep them), as new_device would.  The new trees are built into a new block before the old
 *   block is released, behind the renders still reading it on either pipeline lane, as a prepared scene's update does:
 *   frames enqueued before the update read the old trees, and an update that fails leaves the batch as it was.
 *   Freeing.  ray_b200_scene_batch_free releases the block behind the renders in flight; it is safe to free a batch
 *   whose frames have not finished.
 *   Members.  ray_b200_scene_batch_member(b, s) returns member s as a new, independent prepared scene (its own device
 *   copy of the arrays, indices made local to it; ray_b200_prepared_upload_bytes 0, as for a scene built from device
 *   memory); it is ordered after the batch's build on the context's stream and outlives updates and the batch itself.
 *   Errors (nonzero return and a message; the context stays usable, and a failed call leaves an existing batch unchanged
 *   and usable): the errors of ray_b200_prepare_scene_device and ray_b200_render_into, and n_scenes < 1, B n > 2^26,
 *   B x tiles(h, w) > 2^25 (tiles(h, w) = ceil(h / 4) ceil(w / 8)), a member index outside [0, B), a NULL batch, a shard
 *   set (world > 1), a RAY_GPUS > 1 context, and a host_build context (RAY_HOST_BUILD=1: a batch has no host build). */
struct ray_b200_scene_batch;
int ray_b200_scene_batch_new_device(struct futhark_context *ctx, struct ray_b200_scene_batch **out, int64_t h, int64_t w,
                                    const float *spheres_dev, int32_t n_scenes, int64_t n, const float *cams7_host);
int ray_b200_scene_batch_new_ragged(struct futhark_context *ctx, struct ray_b200_scene_batch **out, int64_t h, int64_t w,
                                    const float *spheres_dev, int32_t n_scenes, const int64_t *counts_host,
                                    const float *cams7_host);
int ray_b200_scene_batch_update(struct futhark_context *ctx, struct ray_b200_scene_batch *b, const float *spheres_dev,
                                const float *cams7_host);
int ray_b200_scene_batch_update_ragged(struct futhark_context *ctx, struct ray_b200_scene_batch *b, const float *spheres_dev,
                                       const int64_t *counts_host /* B counts; may differ from the current ones */,
                                       const float *cams7_host /* NULL keeps the cameras */);
int ray_b200_scene_batch_free(struct futhark_context *ctx, struct ray_b200_scene_batch *b);
/* the batch's B and n (0 when its members' counts differ) */
int ray_b200_scene_batch_shape(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, int32_t *n_scenes,
                               int64_t *n);
/* the batch's B counts */
int ray_b200_scene_batch_counts(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, int64_t *counts_host);
int ray_b200_scene_batch_member(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, int32_t s,
                                struct futhark_opaque_prepared_scene **out);
int ray_b200_render_scene_batch_into(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, int64_t h,
                                     int64_t w, int32_t spp, int32_t *out_pix_dev, float *out_rgb_dev);
/* Ray queries of a scene batch: range sensors, line of sight, shadow rays, picking and depth-complexity lists traced in
 * every scene of a batch in one launch, one entry point for each single-scene ray query ("ray queries" below).  There are
 * m rays per scene: rays_dev is device float[B][m][6] (ranged: struct ray_b200_ray[B][m]), so ray i of the flat array
 * belongs to scene i / m, and the outputs follow the same order: hits_dev struct ray_b200_hit[B][m], rgb_dev
 * float[B][m][3], segments_dev int32[B][m] (or NULL), occluded_dev uint8_t[B][m], multi-hit hits_dev
 * struct ray_b200_hit[B][m][k] and counts_dev int32[B][m] (or NULL); record offsets are 64-bit.  A caller with fewer rays
 * in some scenes pads them with ranged rays whose interval is empty, such as (0, 0): they get the empty answer.
 *   Exactness.  The answer for ray j of scene b is bit for bit what the single-scene entry point returns for that ray on
 *   ray_b200_scene_batch_member(b), and so on ray_b200_prepare_scene_device of scene b's records: every word of every
 *   hit record (sphere is the index into scene b's own records, in [0, n_b)), the colours including their NaNs, segments,
 *   occluded and counts.  Every interval rule of the single-scene queries holds as it is (epsilon 0.1 and the
 *   re-intersection of trace_hits, no epsilon for occlusion and multi-hit, (0, 1e9) for paths, the empty answer for an
 *   invalid per-ray interval).
 *   One launch.  Each call is one launch of the warp-queue kernel over the B m rays, each ray traced from its own scene's
 *   root, planned over all B trees together; asynchronous on the context's stream.  ray_b200_context_last_plan reports
 *   RAY_B200_QUERY_SCENE_BATCH_CLOSEST (hits and paths), _ANYHIT or _MULTIHIT, with n_inner and n_leaves the batch's
 *   totals; last_render_ms and launch_count count it as a single-scene query.  A shard setting is ignored.
 *   Updates and freeing.  A query enqueued before ray_b200_scene_batch_update reads the old trees, one enqueued after it
 *   the new ones; the batch may be freed while a query that reads it is in flight.
 *   Errors (nonzero return and a message; the context stays usable): those of the single-scene query (a non-finite
 *   interval or t_min < 0 in the per-call forms, max_depth outside [0, 65535], k outside [1, 64], a NULL buffer with
 *   m > 0), and a NULL or invalid batch, m < 0 and B m > 2^30.  m == 0 does nothing; max_depth == 0 writes zeros without
 *   a launch. */
struct ray_b200_hit;
struct ray_b200_ray;
int ray_b200_scene_batch_trace_hits(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                    int64_t m, float t_min, float t_max, struct ray_b200_hit *hits_dev);
int ray_b200_scene_batch_trace_paths(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                     int64_t m, int32_t max_depth, float *rgb_dev, int32_t *segments_dev);
int ray_b200_scene_batch_trace_occluded(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, const float *rays_dev,
                                        int64_t m, float t_min, float t_max, uint8_t *occluded_dev);
int ray_b200_scene_batch_trace_multi_hits(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                          const float *rays_dev, int64_t m, float t_min, float t_max, int32_t k,
                                          struct ray_b200_hit *hits_dev, int32_t *counts_dev);
int ray_b200_scene_batch_trace_hits_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                           const struct ray_b200_ray *rays_dev, int64_t m, struct ray_b200_hit *hits_dev);
int ray_b200_scene_batch_trace_occluded_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                               const struct ray_b200_ray *rays_dev, int64_t m, uint8_t *occluded_dev);
int ray_b200_scene_batch_trace_multi_hits_ranged(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                                 const struct ray_b200_ray *rays_dev, int64_t m, int32_t k,
                                                 struct ray_b200_hit *hits_dev, int32_t *counts_dev);

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
 *   Sample s is sample s of the spp semantics above, whatever the chunking.  A call's sample offsets take host and device
 *   memory in proportion to s_end - s_begin, wherever the range starts.
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
/* Adaptive progressive rendering: n_add more samples for the pixels the caller selects, each pixel continuing from its
 * own sample count, so that a progressive renderer spends its samples where the image is still noisy (edges,
 * reflections) and leaves converged pixels alone.
 * accum_dev: device float[h][w][3], row-major: each pixel's running sum.  counts_dev: device int32[h][w]: how many samples
 * that sum holds; where counts[p] == 0 the sum is not read (as at s_begin == 0 above).  mask_dev: device uint8[h][w] (a
 * torch.bool buffer works): a nonzero byte selects the pixel; NULL selects every pixel.
 *   A selected pixel p with c = counts[p] gets samples [c, c + n_add) added to accum[p] one at a time in sample order in
 *   f32 (when c == 0 the sum starts as colour_0 itself), counts[p] becomes c + n_add, and out_pix_dev[p] / out_rgb_dev[p]
 *   (each may be NULL; int32[h][w] / float[h][w][3]) get the pixel at spp = c + n_add: the sum scaled by 1/(c + n_add),
 *   quantised by the rule above.  Sample s is sample s of the spp semantics above, whatever the chunking.
 *   Unselected pixels: none of accum, counts, out_pix or out_rgb is read or written there, so the output frame can be the
 *   caller's persistent display buffer.  A selected pixel whose count is negative, or would pass INT32_MAX (c > INT32_MAX
 *   - n_add), is treated as unselected and left untouched: the library cannot check counts without a device
 *   synchronisation (as invalid intervals of the *_ranged queries give the empty answer).
 *   Exactness: after any sequence of calls on counts that started at 0, accum[p] equals bit for bit what
 *   ray_b200_render_accumulate(s_begin = 0, s_end = counts[p]) leaves at p, and the pixel and float pixel equal
 *   ray_b200_render_into(spp = counts[p]) at p (NaN-aware: a NaN is some NaN).  With mask NULL (or all ones) and every
 *   count equal to s_begin, the call equals ray_b200_render_accumulate(s_begin, s_begin + n_add) in accum and both
 *   outputs, and raises every count by n_add.
 *   The call is asynchronous on the context's stream and is two kernel launches, both counted by
 *   ray_b200_context_launch_count: a selection pass that lists the selected pixels, then the render kernel, which traces
 *   only those (ray_b200_context_last_render_ms covers both).  Stream order and freeing the prepared scene while the call
 *   is in flight behave as for ray_b200_render_accumulate.  It runs on the warp-queue kernel whatever RAY_KERNEL or the
 *   context's kernel says, and uses neither the heavy-first probe nor the learned claim order, nor changes them: renders
 *   before and after it plan and launch exactly as without it.  The selection list (4 bytes per padded pixel) is
 *   stream-ordered device memory freed behind the launch.
 *   Errors (nonzero return, futhark_context_get_error; the context stays usable): every error of
 *   ray_b200_render_accumulate (image size, an invalid prepared scene, a RAY_GPUS > 1 context), n_add < 1,
 *   accum_dev == NULL, counts_dev == NULL, and a shard set (world > 1). */
int ray_b200_render_adaptive(struct futhark_context *ctx, float *accum_dev, int32_t *counts_dev,
                             const uint8_t *mask_dev, int64_t h, int64_t w, int32_t n_add,
                             int32_t *out_pix_dev, float *out_rgb_dev,
                             const struct futhark_opaque_prepared_scene *p);
/* Adaptive progressive rendering with a noise estimate: ray_b200_render_adaptive that also keeps, per pixel and channel,
 * the spread of the pixel's samples, so that a caller can tell where the image is still noisy (ray_b200_adaptive_select).
 * m2_dev: device float[h][w][3], row-major like accum_dev: M2, Welford's running f32 sum of squared deviations from the
 * mean.  Everything ray_b200_render_adaptive promises holds unchanged (selection, counts, outputs, untouched unselected
 * pixels, invalid counts, errors, the two launches); m2 is read and written exactly where accum is.
 *   The rule, per channel: let x_k be the colour of the pixel's sample k, counted over the pixel's whole life, and S_k
 *   the f32 sum of samples [0, k) that accum holds (S_1 = x_0, S_{k+1} = S_k + x_k).  After sample 0, M2 = +0.0 (where
 *   the count is 0, m2 is not read, as accum is not).  Sample k >= 1 updates
 *       M2 = M2 + (x_k - S_k / f32(k)) * (x_k - S_{k+1} / f32(k + 1))
 *   in f32 with IEEE division and no contraction, one sample at a time in sample order, whatever the chunking of calls.
 *   Then M2 / (n - 1) is the sample variance of the pixel's n samples.  Welford's form, not a sum of squares: M2 / n -
 *   mean^2 cancels catastrophically in f32 once counts reach the hundreds.
 *   Exactness: after any sequence of calls on counts that started at 0, accum, counts and both outputs equal what the
 *   same sequence of ray_b200_render_adaptive calls leaves, bit for bit, and m2[p] equals the rule applied to samples
 *   [0, counts[p]) of p (NaN-aware).  Where the caller mixes in other calls, m2 is whatever the caller left there.
 *   Errors: those of ray_b200_render_adaptive, and m2_dev == NULL. */
int ray_b200_render_adaptive_var(struct futhark_context *ctx, float *accum_dev, float *m2_dev, int32_t *counts_dev,
                                 const uint8_t *mask_dev, int64_t h, int64_t w, int32_t n_add,
                                 int32_t *out_pix_dev, float *out_rgb_dev,
                                 const struct futhark_opaque_prepared_scene *p);
/* The pixels of an adaptive progressive frame that still need samples, by the noise estimate of
 * ray_b200_render_adaptive_var: writes mask_dev[p] (device uint8[h][w]; a torch.bool buffer works) = 0 or 1 for every
 * pixel.  With n = counts_dev[p], S = accum_dev[p] and M = m2_dev[p] (device buffers laid out as for
 * ray_b200_render_adaptive_var), mask[p] = 1 iff 0 <= n < max_count and either n < min_count or E > T, where, in f32 and
 * in this order:
 *       v = (M.r + M.g) + M.b
 *       E = v / (f32(n) * f32(n - 1))                  (the three channels' variances of the mean, summed)
 *       m = ((S.r + S.g) + S.b) / f32(n) + mean_floor
 *       T = (rel_err * m) * (rel_err * m)
 *   So a pixel is done when the standard error of its channel sum is at most rel_err times its mean (plus mean_floor,
 *   which keeps dark pixels from asking for a relative error of 0).  NaN compares false: a NaN pixel at or above
 *   min_count is not selected.  accum and m2 are read only where min_count <= n < max_count.  n_selected_dev (device
 *   int32, may be NULL) receives the number of ones.
 *   The call is one kernel launch on the context's stream, asynchronous, counted by ray_b200_context_launch_count; it
 *   leaves ray_b200_context_last_plan and ray_b200_context_last_render_ms unchanged.  The mask feeds the next
 *   ray_b200_render_adaptive_var, so a caller renders "to 1 % noise, at most 512 spp" reading nothing but n_selected:
 *       render_adaptive_var(mask = NULL, n_add = min_spp)
 *       repeat: adaptive_select(..., max_count = max_spp - step + 1, ...); render_adaptive_var(mask, step)
 *   Errors (nonzero return, futhark_context_get_error; the context stays usable): an image size ray_b200_render_into
 *   rejects, a NULL accum_dev, m2_dev, counts_dev or mask_dev, rel_err or mean_floor not finite or below 0,
 *   min_count < 2 (E needs two samples), and max_count < min_count. */
int ray_b200_adaptive_select(struct futhark_context *ctx, const float *accum_dev, const float *m2_dev,
                             const int32_t *counts_dev, int64_t h, int64_t w, float rel_err, float mean_floor,
                             int32_t min_count, int32_t max_count, uint8_t *mask_dev, int32_t *n_selected_dev);
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
/* The first-hit buffers of a frame ("G-buffer", "AOVs"): what each pixel's camera rays hit first, for a denoiser's guide
 * buffers (albedo, normal) and for compositing (depth, sphere id for picking and masks, coverage for alpha at edges).
 * Every output is optional (NULL = not written) and device memory, row-major: id_dev int32[h][w], depth_dev float[h][w],
 * normal_dev and albedo_dev float[h][w][3], coverage_dev int32[h][w].  Offsets are 64-bit.
 *   The rule, for pixel (row j, column i) and sample s in [0, spp): r_s is the camera ray ray_b200_render_into(h, w, spp)
 *   traces on this prepared scene (the prepared camera with this call's pixel grid and the spp semantics above).  H_s is
 *   the struct ray_b200_hit that ray_b200_trace_hits(p, r_s, t_min = 0, t_max = 1e9) returns: objs_hit as ray_colour's
 *   first segment calls it (ray.fut:130), epsilon 0.1 in the search, then re-intersection with (0, t_best + 1), where a
 *   failed re-intersection is no hit.  hit_s means H_s.sphere >= 0.  Then
 *       id       = H_0.sphere (-1 on a miss)
 *       depth    = H_0.t (-1 on a miss), in units of the ray's direction: camera directions are not unit length, and the
 *                  hit point is o + t * d of sample 0's camera ray (which is why there is no position buffer)
 *       coverage = the number of samples s with hit_s
 *       normal   = the mean of x_s = H_s.normal (0 on a miss)
 *       albedo   = the mean of x_s = the colour of sphere H_s.sphere (as ray_b200_scene_get_arrays returns it) where
 *                  hit_s, else the sky colour ray_colour returns for r_s (ray.fut:141-148, light 1), which is
 *                  ray_b200_trace_paths(p, r_s, max_depth = 1)'s colour
 *   A mean is the f32 sum of x_0, ..., x_{spp-1} per component, one sample at a time in sample order, starting from x_0
 *   itself (not 0 + x_0), scaled as the float framebuffer scales a colour sum: the sum itself at spp = 1, else
 *   (1.0f / spp) times the sum.  NaN-aware as elsewhere: a NaN is some NaN.
 *   Identities: id and depth equal ray_b200_trace_hits on sample 0's camera ray; where coverage == 0, albedo equals
 *   ray_b200_render_into(h, w, spp)'s float framebuffer bit for bit (every path there ends in the sky at its first
 *   segment, with light 1); at spp = 1, coverage == (id >= 0).
 *   The call is one kernel launch on the context's stream, asynchronous, counted by ray_b200_context_launch_count and
 *   timed by ray_b200_context_last_render_ms; ray_b200_context_last_plan reports query RAY_B200_QUERY_GBUFFER.  The
 *   prepared scene may be freed or re-uploaded while the call is in flight, as for ray_b200_render_into.  It runs on the
 *   warp-queue kernel whatever RAY_KERNEL or the context's kernel says, each pixel's samples in one slot (never spread),
 *   and uses neither the heavy-first probe nor the learned claim order, nor changes them: renders before and after it
 *   plan and launch exactly as without it.  The buffers converge in a few samples and do not change while a progressive
 *   or adaptive colour frame refines, so a caller computes them once, apart from the colour frame.
 *   Errors (nonzero return, futhark_context_get_error; the context stays usable): every error of ray_b200_render_into
 *   (image size, spp, an invalid prepared scene, a RAY_GPUS > 1 context), all five outputs NULL, and a shard set
 *   (world > 1). */
int ray_b200_render_gbuffer(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                            int64_t h, int64_t w, int32_t spp,
                            int32_t *id_dev, float *depth_dev, float *normal_dev, float *albedo_dev,
                            int32_t *coverage_dev);
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

/* ---- proximity queries: the spheres within a radius of a point, nearest first ----------------------------------------
 * What is near this point: collision candidates of a sphere (the query is the sphere itself), the neighbours of an agent
 * within a radius, how many spheres are within a radius (density, "is this spot free"), the closest sphere surface to a
 * probe point.  A query is a ball (centre c, radius r).  For a sphere with centre p and radius rho (the record layout of
 * ray_b200_scene_from_arrays), the distance is, in f32, in exactly this order, without contraction (IEEE sqrt):
 *     dx = p.x - c.x;  dy = p.y - c.y;  dz = p.z - c.z
 *     d  = sqrtf((dx*dx + dy*dy) + dz*dz) - rho
 * d is the signed distance from c to the sphere's surface (negative when c is inside it), and the sphere is within the
 * ball when d <= r; for a ball that is another sphere's (centre, radius) that means the two touch or overlap.
 *   Answer.  W(i), the set of the scene's spheres within ball i, exactly as a brute force over every sphere computes it.
 *   Unlike the ray queries this does not follow the reference's culling by stale boxes: the walk reads boxes that contain
 *   their subtrees (for a scene with stale boxes they are rebuilt first, see below) with a ball-box test that is
 *   conservative by a proved margin (DESIGN.md §5d), and every sphere it reaches is tested by the rule above.  A sphere
 *   whose radius is negative or NaN (-0.0 is a valid point sphere), or with a non-finite centre component or radius, is
 *   never reported.  A ball whose centre is not finite, or whose r is not finite and >= 0, gets the empty answer; it is
 *   not an error (the host does not read the balls), and the other balls are unaffected.
 *   Outputs.  counts_dev[i] = |W(i)|, not capped at k (device int32[n], or NULL).  near_dev[i][j], j < min(k, |W(i)|):
 *   the j-th member of W(i) as struct ray_b200_near, ordered by ascending d, then ascending caller index; d is never -0.0
 *   (it is x - rho rounded to nearest); the remaining records are d = +inf, sphere = -1 (device struct ray_b200_near[n][k],
 *   record offsets are 64-bit; NULL is allowed when k == 0, the count-only query).
 *   Stale boxes.  A scene whose stored boxes are all the union of their children's (ray_b200_prepared_info's stale_nodes
 *   == 0) is walked as it is stored.  Otherwise each call first builds complete boxes (the refit run to its fixpoint) into
 *   scratch the context owns, grown on demand and freed with the context: a copy of the records, two memsets and two
 *   more launches.  The prepared scene is not changed.
 *   Calls.  Asynchronous on the context's stream; balls_dev is read after the work enqueued there before the call.  One
 *   launch, plus two for a scene with stale boxes, all counted by ray_b200_context_launch_count; last_plan and
 *   last_render_ms are unchanged (this is not a warp-queue launch).  A prepared scene or batch may be freed or updated
 *   while a query that reads it is in flight.  On a RAY_GPUS > 1 context the query runs on device d, which holds the scene.
 *   Errors (nonzero return, futhark_context_get_error; nothing is written and the context stays usable): n outside
 *   [0, 2^30], k outside [0, 64], a NULL balls_dev, a NULL near_dev with k > 0, k == 0 with a NULL counts_dev (no output),
 *   and an invalid prepared scene.  n == 0 does nothing.
 *   Scene batches.  ray_b200_scene_batch_query_spheres takes m balls per scene: balls_dev struct ray_b200_ball[B][m],
 *   near_dev struct ray_b200_near[B][m][k], counts_dev int32[B][m], uniform or ragged.  The answer for ball j of scene b is
 *   bit for bit the single-scene answer on ray_b200_scene_batch_member(b): sphere indexes scene b's own records.  Complete
 *   boxes are built for the whole batch when any member has stale boxes.  Further errors: a NULL or invalid batch, m < 0
 *   and B m > 2^30. */
struct ray_b200_ball {
  float c[3];   /* centre */
  float r;      /* radius of the query */
};              /* 16 bytes, 4-byte aligned */
struct ray_b200_near {
  float d;          /* signed distance from the ball's centre to the sphere's surface; +inf for an unused record */
  int32_t sphere;   /* index into the scene's sphere array as given; -1 for an unused record */
};                  /* 8 bytes */
int ray_b200_query_spheres(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           const struct ray_b200_ball *balls_dev, int64_t n, int32_t k, struct ray_b200_near *near_dev,
                           int32_t *counts_dev);
int ray_b200_scene_batch_query_spheres(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                       const struct ray_b200_ball *balls_dev, int64_t m, int32_t k,
                                       struct ray_b200_near *near_dev, int32_t *counts_dev);
/* sizeof(struct ray_b200_near) (8) and sizeof(struct ray_b200_ball) (16) as the library was compiled. */
int64_t ray_b200_near_size(void);
int64_t ray_b200_ball_size(void);

/* ---- nearest-sphere queries: the k nearest spheres to a point, with no radius to guess -----------------------------------
 * Which k spheres are nearest to this point, however far away: the signed distance of the scene at a probe point (sphere
 * tracing, collision margins, training data for distance fields), the k-nearest-neighbour graph of the spheres
 * themselves, the closest object to a cursor.  A query is a struct ray_b200_ball (c, r) whose r is an upper limit on d,
 * r = +inf for no limit.  d is the proximity queries' distance above, in f32 in the same operation order, and the same
 * spheres are reportable (finite centre and radius, rho >= 0, -0.0 included).
 *   Balls.  A ball is valid when its centre is finite and r >= 0, r = +inf included; a ball with a non-finite centre, or
 *   whose r is NaN or negative, gets the empty answer.  That is not an error, and the other balls are unaffected.  This
 *   differs from ray_b200_query_spheres only in accepting r = +inf (query_spheres still gives such a ball the empty answer).
 *   Answer.  W(i), the reportable spheres with d <= r_i.  near_dev[i][j] for j < min(k, |W(i)|) is the j-th member of
 *   W(i) in ascending d, then ascending caller index (query_spheres' order); the remaining records are d = +inf,
 *   sphere = -1 (device struct ray_b200_near[n][k], record offsets are 64-bit).  With r = +inf a reportable sphere's d may
 *   overflow to +inf: it is still a record, with sphere >= 0, so `sphere` tells a record from padding.  There is no count:
 *   ray_b200_query_spheres counts the spheres within a bounded r.
 *   Identities.  For a finite r the records are bit for bit ray_b200_query_spheres(ball, k)'s.  At k = 1, record 0's d is
 *   the signed distance at c of the union of the scene's reportable spheres (min over them of |p - c| - rho), or +inf
 *   when there are none.
 *   Neighbour graph.  The k nearest other spheres of sphere i: query its own centre with k + 1 (r = +inf, or a limit) and
 *   drop the record with sphere == i, or the last record when i is absent; that is exactly the first k of W minus {i},
 *   whatever coincident copies do to the order.  As k is at most 64, this gives at most 63 neighbours.
 *   Stale boxes, calls.  As for ray_b200_query_spheres: a scene with stale boxes is walked over complete boxes built into
 *   the context's scratch first (the prepared scene is not changed); asynchronous on the context's stream, balls_dev read
 *   after the work enqueued there before the call; one launch, plus two for a scene with stale boxes, all counted by
 *   ray_b200_context_launch_count; last_plan and last_render_ms are unchanged.  A prepared scene or batch may be freed or
 *   updated while a query that reads it is in flight.  On a RAY_GPUS > 1 context the query runs on device d.
 *   Errors (nonzero return, futhark_context_get_error; nothing is written and the context stays usable): n outside
 *   [0, 2^30], k outside [1, 64], a NULL balls_dev or near_dev with n > 0, an invalid prepared scene.  n == 0 does
 *   nothing.
 *   Scene batches.  ray_b200_scene_batch_query_nearest takes m balls per scene: balls_dev struct ray_b200_ball[B][m],
 *   near_dev struct ray_b200_near[B][m][k], uniform or ragged; ball j of scene b gets the single-scene answer on
 *   ray_b200_scene_batch_member(b), sphere indexing scene b's own records.  Further errors: a NULL or invalid batch, m < 0
 *   and B m > 2^30. */
int ray_b200_query_nearest(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                           const struct ray_b200_ball *balls_dev, int64_t n, int32_t k,
                           struct ray_b200_near *near_dev);
int ray_b200_scene_batch_query_nearest(struct futhark_context *ctx, const struct ray_b200_scene_batch *b,
                                       const struct ray_b200_ball *balls_dev, int64_t m, int32_t k,
                                       struct ray_b200_near *near_dev);

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
