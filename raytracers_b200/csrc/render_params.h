// Kernel parameter block shared by the host API (api.cu) and the kernels (render_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/ray_b200.h"   // enum ray_b200_kernel (LaunchConfig::kernel)

namespace rayb200 {

constexpr int kTileW = 8;       // a warp renders an 8x4-pixel tile (coherent primary rays, 128-B stores)
constexpr int kTileH = 4;
constexpr int kTilePixels = 32;
constexpr int kMaxDepth = 50;   // ray.fut:154 `ray_colour objs ray 50`
constexpr int kStackSize = 64;  // a radix tree over (32-bit key, 32-bit index) is at most 64 deep

struct RenderParams {
  // prepared scene (device layout of scene_host.h PackedBvh)
  const float4 *nodes;      // node-major records (global fetch path)
  const float4 *nodes_soa;  // component-major copy (source of the shared-memory staging)
  const float4 *geom;
  const float4 *colour;
  int32_t n_inner, n_leaves;
  int32_t smem_nodes;    // first smem_nodes BFS nodes are staged in shared memory (every kernel but K0)
  int32_t smem_spheres;  // first smem_spheres sphere records staged (0 or n_leaves)
  int32_t max_depth;     // depth of the deepest leaf (root = 0): bounds the traversal stacks
  float root_box[6];
  float cam[12];         // origin, llc, horizontal, vertical (ray.fut:88-91)
  // frame
  int32_t W, H, spp;
  float inv_spp;
  const float *offsets;  // 2*spp sample offsets of the launch's samples (device; a chunk's start at its s_begin)
  int32_t *out_pix;      // row-major [H][W] (tile_major == 0) or compact [local_tiles][32] (tile_major == 1)
  float *out_rgb;        // optional [H][W][3]
  int32_t tile_major;
  // sharding: this rank renders tiles t = lt * world + rank
  int32_t rank, world, tiles_x, tiles_y;
  int64_t n_tiles, local_tiles;
  // claim order of the persistent kernels: work is claimed in chunks of 64 tiles (2048 pixels) and the
  // chunk order is a stride permutation (chunk * chunk_stride mod n_chunks, stride coprime to n_chunks), so
  // the cheap sky and the 50-bounce ground of a frame are interleaved instead of the heavy rows coming last
  int32_t n_chunks, chunk_stride;
  // heavy-first claim order (NULL = the chunk permutation above): the same permuted sequence, except that tiles whose
  // probe path is long are pulled into its first half, so that a frame never ends on a 50-bounce path claimed late
  const int32_t *tile_order;
  int32_t chunk_stride_inv;  // chunk_stride * chunk_stride_inv = 1 (mod n_chunks): position of a tile chunk in the claim sequence
  int32_t probes_per_tile, probe_segments;
  // learned claim order: when non-NULL (warp-queue kernel) every finished path records max(segments) of its 8x4 tile here;
  // the next frame of the same prepared scene and geometry claims the tiles with long paths first (api_render.cu)
  uint32_t *tile_cost;
  float4 *sample_buf;    // warp-queue kernel, spp > 1: [CTAs][warps][kWqRing][spp] finished-sample colours (else NULL)
  // persistent-threads work cursor ([0]; [1] counts the warps that have left the kernel when frame_flag is set) and
  // optional work counters
  int32_t *work_cursor;
  // peer-frame protocol (NULL = off): out_pix may be a peer device's frame; the last warp to leave the kernel bumps
  // *frame_flag (system scope) after a system-wide fence, so the consumer knows this rank's pixels have landed
  uint32_t *frame_flag;
  unsigned long long *counters;  // [4] segments, node_steps, box_tests, leaf_tests (counting kernels only)
  // diagnostic (NULL unless tracing): [0] = earliest CTA start, [1 + cta * warps + warp] = that warp's exit, in
  // %globaltimer ns — shows how long the SMs sit idle behind the frame's last paths (warp-queue kernel only)
  unsigned long long *warp_trace;
};

// What the warp-queue kernel traces (its template parameter kQuery), and which RayQuery fields the launch reads.
// Pixel kinds, camera rays: kPixels, a whole frame (no field); kAccumulate, one chunk of a progressive frame (accum,
// s_begin); kViews, several views in one launch (cams, n_views, view_tiles).  Ray kinds, the caller's rays of a ray query
// (include/ray_b200.h "ray queries"; rays, n, perm, t_min, t_max): kClosest, to their closest hit (hits) or along their
// path (rgb, segments, max_depth; hits == NULL tells the two apart at run time); kAnyHit, to their first accepted sphere
// (occluded); kMultiHit, to their k nearest ones (hits, k, counts).  kAdaptive, a pixel kind: the selected pixels of a
// progressive frame, each from its own sample count (accum, sample_counts, mask, sel, n_sel).  kAdaptiveVar: kAdaptive
// that also keeps each pixel's running sum of squared deviations (m2).  kGBuffer, a pixel kind: the first hit of every
// camera ray of a frame (its sphere, t, normal and albedo), reduced per pixel into the guide buffers (gb_id, gb_depth,
// gb_normal, gb_albedo, gb_coverage).  kSceneBatch, a pixel kind: one frame of each scene of a scene batch (cams, n_views,
// view_tiles as kViews, root_boxes, scene_off).  kBatchClosest, kBatchAnyHit and kBatchMultiHit, ray kinds: the
// single-scene ray kind over the trees of a scene batch, rays_per_scene rays per scene (root_boxes, scene_off as
// kSceneBatch).  New kinds go at the end: kernel names carry the values, and tools/sass_compare.py reads older builds'
// names by them.
enum class Query { kPixels, kClosest, kAnyHit, kMultiHit, kAccumulate, kViews, kAdaptive, kAdaptiveVar, kGBuffer, kSceneBatch,
                   kBatchClosest, kBatchAnyHit, kBatchMultiHit };
// The ray kinds of a scene batch
__host__ __device__ constexpr bool is_batch_ray(Query q) {
  return q == Query::kBatchClosest || q == Query::kBatchAnyHit || q == Query::kBatchMultiHit;
}
// What a launch of kind q computes per ray or pixel: a scene batch's ray kind is its single-scene kind, every other kind
// itself.  The kernel tests this, not q, for what the single-scene ray kinds do, so that each is named once.
__host__ __device__ constexpr Query single_scene_kind(Query q) {
  return q == Query::kBatchClosest ? Query::kClosest
       : q == Query::kBatchAnyHit ? Query::kAnyHit
       : q == Query::kBatchMultiHit ? Query::kMultiHit : q;
}
__host__ __device__ constexpr bool is_ray_query(Query q) {
  const Query s = single_scene_kind(q);
  return s == Query::kClosest || s == Query::kAnyHit || s == Query::kMultiHit;
}
// Pixel kinds whose pixels each continue from their own sample count (Q.sample_counts): a selection pass in front of the
// render kernel lists the pixels, which the kernel claims from Q.sel; each sample's offsets are computed on the device, so
// no offset table is made
__host__ __device__ constexpr bool is_adaptive(Query q) { return q == Query::kAdaptive || q == Query::kAdaptiveVar; }
// Pixel kinds that continue a pixel's running sum in Q.accum and store it back.  Such a launch uses neither the heavy-first
// probe nor the learned claim order, and leaves the learned order as it found it.
__host__ __device__ constexpr bool is_progressive(Query q) { return q == Query::kAccumulate || is_adaptive(q); }
// Pixel kinds whose slots always own their pixel, whatever the sample count: the launch gets no finished-sample buffer,
// so it is planned and launched as a pixel-bound frame
__host__ __device__ constexpr bool is_pixel_bound(Query q) { return q == Query::kGBuffer; }
// Pixel kinds that claim the frame's tiles in the plain chunk permutation: a launch uses neither the heavy-first probe
// nor the learned claim order, and leaves the learned order as it found it
__host__ __device__ constexpr bool is_plain_order(Query q) { return is_progressive(q) || q == Query::kGBuffer || q == Query::kSceneBatch; }
// Pixel kinds whose work items are the tiles of several frames, one after the other (RayQuery::view_tiles each), each
// frame drawn with its own camera of RayQuery::cams and written at its own offset
__host__ __device__ constexpr bool is_multi_frame(Query q) { return q == Query::kViews || q == Query::kSceneBatch; }

// The fields of a launch that RenderParams does not carry (see Query for which kind reads which).  A block of its own,
// passed after the kernel's scalar parameters: new fields at the end of RenderParams would move those parameters, and
// with them the constant-bank offsets in every pixel instantiation's code.
struct RayQuery {
  const float *rays;        // [n][6]: origin.xyz, dir.xyz; ranged query: [n][8] = struct ray_b200_ray
  float *rgb;               // path query: [n][3] colour of ray_colour (ray.fut:126-148)
  int32_t *segments;        // path query, optional: [n] objs_hit calls of the path
  float *hits;              // hit query (non-NULL = hit mode): [n][8] struct ray_b200_hit; multi-hit query: [n][k][8]
  const int32_t *perm;      // Morton-sorted leaf -> index into the caller's sphere array
  int32_t n;
  float t_min, t_max;       // hit / occlusion / multi-hit query: the call's interval (unused when ranged: each ray has
                            // its own); path query: (0, 1e9) as ray_colour passes it
  int32_t max_depth;        // path query: the depth limit of ray_colour (1 for the one-segment queries)
  uint8_t *occluded;        // occlusion query: [n] 0 / 1
  int32_t k;                // multi-hit query: records per ray, in [1, 64]
  int32_t *counts;          // multi-hit query, optional: [n] accepted leaves per ray, not capped at k
  // progressive rendering (Query::kAccumulate; include/ray_b200.h ray_b200_render_accumulate): the frame's samples
  // [s_begin, s_begin + P.spp) are added to accum, row-major [H][W][3], the running f32 sum of each pixel's samples
  // [0, s_begin) (not read when s_begin == 0)
  float *accum;
  int32_t s_begin;
  // several views of one prepared scene (Query::kViews; include/ray_b200.h ray_b200_render_views_into): n_views frames
  // of P.W x P.H, one after the other.  Work-item tiles [v * view_tiles, (v + 1) * view_tiles) are view v's tiles in the
  // row-major tile order of one frame; view v is drawn with the camera cams[v] (device [n_views][12], 16-byte aligned,
  // laid out as RenderParams::cam) and written at pixel offset v * H * W of the outputs
  const float *cams;
  int32_t n_views, view_tiles;
  // adaptive progressive rendering (Query::kAdaptive; include/ray_b200.h ray_b200_render_adaptive): P.spp = n_add samples
  // are added to the selected pixels, each from its own count.  sample_counts, row-major [H][W]: the samples in accum's
  // sum of each pixel (accum is not read where it is 0); mask, row-major [H][W] (NULL = every pixel): nonzero = selected.
  // The selection pass writes the work items of the selected pixels with a valid count to sel, in claim order, and their
  // number to *n_sel, which the render kernel claims instead of the frame's tiles
  int32_t *sample_counts;
  const uint8_t *mask;
  int32_t *sel;
  int32_t *n_sel;
  // Query::kAdaptiveVar (include/ray_b200.h ray_b200_render_adaptive_var): row-major [H][W][3], each pixel's M2, Welford's
  // running f32 sum of squared deviations from the mean of its samples (not read where its count is 0)
  float *m2;
  // Query::kGBuffer (include/ray_b200.h ray_b200_render_gbuffer): the guide buffers of the frame, row-major, each optional
  // (NULL = not written): [H][W] sphere id and t of sample 0's first hit, [H][W][3] mean normal and albedo of the first
  // hits, [H][W] samples whose camera ray hit a sphere
  int32_t *gb_id;
  float *gb_depth;
  float *gb_normal;
  float *gb_albedo;
  int32_t *gb_coverage;
  // a scene batch (Query::kSceneBatch; include/ray_b200.h ray_b200_render_scene_batch_into): n_views = B frames as kViews
  // lays them out, frame b of scene b with the camera cams[b].  The B trees lie back to back in P's arrays with global
  // indices: scene b's leaves start at scene_off[b] (device [B + 1]) and its inner nodes at scene_off[b] - b, so its root
  // is node scene_off[b] - b; its root box is the first 6 floats of root_boxes[8 b .. 8 b + 8) (struct BvhBuildResult
  // records, 32-byte aligned), tested at every segment's set-up instead of P.root_box
  const float *root_boxes;
  const int32_t *scene_off;
  // the ray kinds of a scene batch (Query::kBatchClosest / kBatchAnyHit / kBatchMultiHit; include/ray_b200.h
  // ray_b200_scene_batch_trace_*): rays [b * rays_per_scene, (b + 1) * rays_per_scene) are scene b's, traced from its root
  // node and root box as kSceneBatch; n = B * rays_per_scene, and the outputs follow the rays' order
  int32_t rays_per_scene;
};

// Wavefront ray queues (SoA in HBM, 48 B per live ray): two ping-pong queues indexed by bounce parity.
struct WavefrontBuffers {
  float4 *ray_o[2];   // {origin.xyz, bits(path id = local item index)}
  float4 *ray_d[2];   // {dir.xyz, 0}
  float4 *light[2];   // {light.rgb, 0}
  int32_t *qlen;      // [kMaxDepth + 2] rays queued for bounce b (written by bounce b-1's compaction)
  int32_t *cursor;    // [kMaxDepth + 2] persistent-threads work cursor of bounce b
  float4 *accum;      // per local item {sum.rgb, 0}: in-order sample accumulation when spp > 1
  int64_t capacity;   // items the queues can hold
  int32_t tail_from;  // bounce whose kernel runs the (few) surviving rays to completion
  // N4 experiment (ray re-sorting between bounces, DESIGN.md): before bounces 1..sort_bounces the queue is
  // ordered by (direction octant, Morton code of the origin in the root box) through an index array
  int32_t sort_bounces;
  uint32_t *sort_keys, *sort_keys_out;  // [capacity]
  int32_t *sort_ids, *order;            // [capacity]; order[i] = queue entry to be traced i-th
  void *sort_tmp;
  size_t sort_tmp_bytes;
};
size_t wavefront_sort_bytes(int64_t items);  // cub temp storage for the re-sort (0 in builds without the alternative kernels)

// The launch plan of one frame or ray query: fill_params returns it next to the RenderParams (trace() in api_rays.cu makes
// the ray queries'), and the launcher of its kernel reads only the fields that kernel uses.
struct LaunchConfig {
  int kernel;          // ray_b200_kernel
  int blocks_per_sm;
  int sm_count;
  int refill_min;      // persistent kernel: refill when at least this many lanes are idle
  int wq_warps;        // warp-queue / stream-queue / lane-walk kernels: warps per CTA (one CTA per SM)
  int wq_k;            // warp-queue kernel: rays in flight per warp = 32 * wq_k (1 or 2)
  int wq_refill;       // warp-queue / stream-queue kernels, spread mode: hand out samples when at least this many slots are idle
  int wq_low;          // warp-queue kernel: node batches take the OLDEST queued items while at most this many are queued (0 = half the ring, < 0 = never)
  int wq_packet;       // warp-queue kernel: node steps with at least this many lanes are done packet-style (0 = never)
  int wq_ncap;         // warp-queue kernel: cap on the node-queue capacity (0 = the proved bound, at most 1024)
  int lw_slots;        // lane-walk kernel: path slots per warp (32 lanes walk, the rest wait for / come from shading)
  int lw_idle_min;     // lane-walk kernel: with the ready list empty, shade as soon as this many lanes have nothing to walk
  int lw_passes;       // lane-walk kernel: refill passes per shading phase
  int max_dynamic_smem;  // the device's opt-in shared-memory limit (kernels opt in on first launch)
  long long stage_budget;  // warp-queue kernel: shared memory its queues leave for staging, before cap_staging (bytes)
};

// A frame of pixel kind `kind` on the kernel lc.kernel names (render_kernels.cu); every kind but kPixels reads q and runs
// on the warp-queue kernel only
cudaError_t launch_render(const RenderParams &p, const LaunchConfig &lc, const WavefrontBuffers *wf, cudaStream_t stream,
                          int64_t *launches, Query kind, const RayQuery &q);
// The warp-queue kernel (render_kernels.cu): a launch of kind `kind`, a pixel kind or a ray query (whatever lc.kernel
// says); `ranged`: q.rays is [n][8] with an interval per ray (hit, occlusion and multi-hit queries)
cudaError_t launch_warpqueue(const RenderParams &p, Query kind, bool ranged, const RayQuery &q, const LaunchConfig &lc,
                             cudaStream_t stream, int64_t *launches);
// per translation unit: K5 (render_lanewalk.cu) and the alternatives K1 / K2 / K4 (render_alt_kernels.cu; a product
// build without RAYB200_ALL_KERNELS returns cudaErrorNotSupported)
cudaError_t launch_lanewalk(const RenderParams &p, const LaunchConfig &lc, cudaStream_t stream, int64_t *launches);
cudaError_t launch_alt_kernel(const RenderParams &p, const LaunchConfig &lc, const WavefrontBuffers *wf, cudaStream_t stream,
                              int64_t *launches);
cudaError_t preload_default_kernels(int max_dynamic_smem);  // render_kernels.cu: the variants of the default plan
// Probe pass + sort that produce RenderParams::tile_order (see render_kernels.cu).  All buffers are device memory.
struct TileOrderBuffers {
  uint32_t *keys, *keys_sorted;   // [local_tiles]
  int32_t *ids, *order;           // [local_tiles]
  void *sort_tmp;
  size_t sort_tmp_bytes;
};
size_t tile_order_sort_bytes(int64_t local_tiles);
inline int tile_order_key_bits(int32_t n_chunks) {  // keys are positions < n_chunks * 64
  int bits = 6;
  while (bits < 32 && (1ll << bits) < (long long)n_chunks * 64) bits++;
  return bits;
}
// Query::kAdaptive: the selection pass in front of the render kernel (q.sel, q.n_sel; *q.n_sel zeroed by the caller)
void launch_adaptive_select(const RenderParams &p, const RayQuery &q, cudaStream_t stream, int64_t *launches);
// ray_b200_adaptive_select (include/ray_b200.h): the noise rule over n_px pixels, mask[p] = 0 / 1, and the number of ones
// added to *n_selected where it is not NULL (zeroed by the caller)
void launch_adaptive_error_select(const float *accum, const float *m2, const int32_t *counts, int64_t n_px, float rel_err,
                                  float mean_floor, int32_t min_count, int32_t max_count, uint8_t *mask, int32_t *n_selected,
                                  cudaStream_t stream, int64_t *launches);
// of a frame of pixel kind `kind`: Query::kViews probes each tile with its view's camera (q.cams)
void launch_tile_order(const RenderParams &p, const TileOrderBuffers &b, cudaStream_t stream, int64_t *launches, Query kind,
                       const RayQuery &q);
// The same order table from a recorded frame: tiles whose longest path had >= long_path segments first, both groups in
// the permuted claim sequence (cost = RenderParams::tile_cost of the recorded frame)
void launch_tile_order_from_cost(const RenderParams &p, const uint32_t *cost, int32_t long_path, const TileOrderBuffers &b,
                                 cudaStream_t stream, int64_t *launches);
// peer-frame flags (render_kernels.cu): 1-thread kernels on `stream`
void launch_flag_wait(uint32_t *flag, uint32_t value, long long timeout_ns, unsigned long long *timeouts, cudaStream_t stream);
void launch_flag_set(uint32_t *flag, uint32_t value, cudaStream_t stream);
void launch_flag_bump(uint32_t *flag, cudaStream_t stream);  // for the kernels that do not signal themselves
void launch_count_work(const RenderParams &p, cudaStream_t stream, int64_t *launches);
void launch_detile(const int32_t *gathered, int32_t *out, int64_t H, int64_t W, int32_t world, int64_t tiles_padded,
                   cudaStream_t stream, int64_t *launches);
// dynamic shared memory of the BVH staging area: [mbarrier, padded to 128 B][nodes][sphere records]
__host__ __device__ inline size_t staging_bytes(const RenderParams &p) {
  return 128 + (size_t)p.smem_nodes * 64 + (size_t)p.smem_spheres * 16;
}
// CTA size bound of the warp-queue kernels = their register budget: 1024 threads -> 64 registers (a few spills in the
// cold paths), 768 -> 80.  32 warps x 64 registers are the default: the kernel is bound by issue slots and latency, not
// registers (sm_90 has the same 64 K registers and 2048 threads per SM as the part this was first tuned on).
#ifndef RAYB200_WQ_THREADS
#define RAYB200_WQ_THREADS 1024
#endif
constexpr int kWqMaxThreads = RAYB200_WQ_THREADS;  // warp-queue kernel: CTA size bound (one CTA per SM) -> register budget
constexpr int kWqMaxWarps = kWqMaxThreads / 32;
constexpr int kWqRing = 8;         // warp-queue kernel: pixels a warp may have open at once when samples are spread
constexpr int kWqLeafStack = 128;  // warp-queue kernel: leaf-item stack (never more than 31 + 64 live)
constexpr int kWqPacketStack = 64; // warp-queue kernel: deferred (node, mask) pairs of the packet walk (<= tree depth)
// warp-queue kernel: node-stack capacity (proved bound, see render_kernels.cu) and per-warp / per-CTA bytes
__host__ __device__ inline int wq_node_capacity(int k, int max_depth) {
  // 32k + 64(depth+1) is the proved bound of the depth-sorted LIFO; the drain loop's overflow guard makes ANY capacity
  // >= 256 safe (it falls back to one-item-at-a-time DFS when fewer than 96 entries are free), so deep trees are
  // capped at 1024 entries instead of costing warps or staging space
  const int c = 32 * k + 64 * (max_depth + 1);
  return c < 256 ? 256 : (c > 1024 ? 1024 : c);
}
// ... optionally capped further (tuning parameter wq_ncap, 0 = no cap): trades queue space for staged BVH nodes
__host__ __device__ inline int wq_node_capacity(int k, int max_depth, int cap) {
  const int c = wq_node_capacity(k, max_depth);
  return cap > 0 && cap < c ? (cap < 256 ? 256 : cap) : c;
}
// (a slot = 4 float4 {origin + a, 1/dir, dir, light + depth} + best t / leaf + item, and per-pixel sample state: a float4
// {sum, sample} when a slot owns a pixel, 4 bytes {ring entry, sample} when samples are spread)
__host__ __device__ inline size_t wq_warp_bytes(int k, int ncap, bool packet, bool spread) {
  const size_t r = 32 * (size_t)k;
  return ((r * (16 * 4 + (spread ? 4 : 16) + 8 + 4) + 2 * kWqRing * 4 + (packet ? 2 * kWqPacketStack * 4 : 0) + kWqLeafStack * 4 + (size_t)ncap * 4) + 127) & ~(size_t)127;
}
// The warp-queue kernel's launch of kind `kind` (`ranged`: per-ray intervals) with parameter block p and plan lc: the
// template flags it instantiates and its launch geometry.  launch_warpqueue launches exactly this, and the context's
// launch report (ray_b200_context_last_plan) is made from it.  ctas == 0: there is no work, nothing is launched.
struct WqVariant {
  int k;                     // rays in flight per warp / 32
  bool spread, packet;       // samples spread over a warp's slots (a finished-sample buffer is set); packet walk
  bool all_nodes, spheres;   // every node staged; every sphere record staged as well
  int ncap, nlow;            // node-queue allocation; breadth-first below nlow queued items
  size_t smem;               // dynamic shared memory of a CTA
  long long ctas;
};
inline WqVariant wq_variant(const RenderParams &p, Query kind, const RayQuery &q, const LaunchConfig &lc) {
  WqVariant v;
  const bool rays = is_ray_query(kind);
  v.spread = !rays && p.sample_buf != nullptr;
  v.packet = !rays && lc.wq_packet > 0;
  v.all_nodes = p.smem_nodes == p.n_inner;
  v.spheres = p.smem_spheres == p.n_leaves && p.smem_spheres > 0;
  v.k = lc.wq_k == 1 ? 1 : 2;
  v.ncap = wq_node_capacity(v.k, p.max_depth, lc.wq_ncap);
  const int nring = 1 << (31 - __builtin_clz((unsigned)v.ncap));
  v.nlow = lc.wq_low < 0 ? 0 : (lc.wq_low == 0 ? nring / 2 : (lc.wq_low > nring - 96 ? nring - 96 : lc.wq_low));
  v.smem = ((staging_bytes(p) + 127) & ~(size_t)127) + (size_t)lc.wq_warps * wq_warp_bytes(v.k, v.ncap, v.packet, v.spread);
  // no more CTAs than there are rays to start at once: a slot takes one query ray, one SAMPLE when samples are spread, one
  // pixel otherwise (capping by pixels alone left 26 SMs idle on a 125 K-pixel shard at 64 spp with 32 warps per CTA)
  const long long work = rays ? (long long)q.n : p.local_tiles * kTilePixels * (v.spread ? (long long)p.spp : 1ll);
  const long long useful = work <= 0 ? 0 : (work + 32 * v.k * lc.wq_warps - 1) / (32 * v.k * lc.wq_warps);
  v.ctas = lc.sm_count < useful ? lc.sm_count : useful;
  return v;
}

// stream-queue kernel (K4): per-warp bytes (5 float4 + best + item + pending per slot, done/free lists, ring, stacks)
__host__ __device__ inline size_t sq_warp_bytes(int k, int ncap) {
  const size_t r = 32 * (size_t)k;
  return ((r * (16 * 5 + 8 + 4 + 4 + 4 + 4) + 2 * kWqRing * 4 + kWqLeafStack * 4 + (size_t)ncap * 4) + 127) & ~(size_t)127;
}


// lane-walk kernel (K5): private DFS stack entries per lane (<= one deferred sibling per level) and per-warp bytes:
// R slots x (4 float4 + best t / leaf + item + meta), sample ring, leaf-item stack, [scap][32] DFS stacks, 3 slot lists
__host__ __device__ inline int lw_stack_capacity(int max_depth) { return max_depth + 1 < 4 ? 4 : max_depth + 1; }
__host__ __device__ inline size_t lw_warp_bytes(int slots, int scap) {
  const size_t r = (size_t)slots;
  return (r * (16 * 4 + 4 * 4) + 2 * kWqRing * 4 + kWqLeafStack * 4 + (size_t)scap * 128 + ((3 * r + 15) & ~(size_t)15) + 127) & ~(size_t)127;
}

}  // namespace rayb200
