// sm_90a render kernels of the product build: K0 (thread per pixel: the parity anchor and the counting kernel), the
// tile probe of the heavy-first claim order, K3 (warp work-queue) and the multi-GPU de-tiling kernel, plus the host
// launchers.  K5 (the lane-walk kernel) is in render_lanewalk.cu, the measured-slower alternatives K1 / K2 / K4 in
// render_alt_kernels.cu (compiled with RAYB200_ALL_KERNELS only).  Shared device code: render_common.cuh.
#include <cub/cub.cuh>
#include "render_common.cuh"

namespace rayb200 {

namespace {

// ====================================================================================== K0: megakernel
// One thread per pixel, the whole ray_colour loop inside (what a Futhark GPU backend would emit,
// SURVEY.md §8a A11).  The parity anchor and the "naive GPU" number.
template <bool kCount>
__global__ void __launch_bounds__(128) render_mega_kernel(const __grid_constant__ RenderParams P) {
  const long long k64 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  WorkCounters wc;
  int i = 0, j = 0;
  const bool valid = k64 < P.local_tiles * kTilePixels && item_pixel(P, (int)k64, i, j);
  if (valid) {
    const GlobalScene sc{P.nodes, P.geom};
    V3 sum = v3(0.0f, 0.0f, 0.0f);
    for (int s = 0; s < P.spp; s++) {
      Ray r = primary_ray(P, i, j, s);
      V3 light = v3(1.0f, 1.0f, 1.0f), colour;
      int depth = 0;
      while (advance_path<kCount>(sc, P, r, light, depth, colour, wc)) {}
      sum = (s == 0) ? colour : vadd(sum, colour);
    }
    write_pixel(P, (int)k64, i, j, sum);
  } else if (P.tile_major && k64 < P.local_tiles * kTilePixels) {
    P.out_pix[k64] = 0;  // padding pixel of a partial tile
  }
  if (kCount) flush_counters(P, wc);
}

// ====================================================================================== heavy-first claim order
// The persistent kernels end a frame on whatever was claimed last; a 50-bounce path claimed late keeps one warp busy
// for ~50 dependent traversals while the other SMs idle.  Sorting the tiles longest-first cures the tail but un-mixes
// the frame — first every warp waits on L2 for deep nodes, then every warp shades sky — and the bulk gets slower.  So the claim order
// stays the chunk permutation, and only the tiles whose probe path is still alive after `probe_segments` segments
// ("heavy": possibly 50 bounces) are pulled into its first half: key = position in the permuted sequence, halved for
// heavy tiles, stable-sorted.  What is claimed in the second half ends within probe_segments traversals.  The probe
// traces sample 0 of 1, 2 or 4 pixels per 8x4 tile, so its own latency is bounded by the same cap.  The order only
// changes WHEN a pixel is rendered, never its value.
__global__ void __launch_bounds__(256) tile_probe_kernel(const __grid_constant__ RenderParams P, uint32_t *__restrict__ keys,
                                                         int32_t *__restrict__ ids) {
  const int probes = P.probes_per_tile;  // 1, 2 or 4: the lanes of a tile are neighbours in a warp
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long lt = t / probes;
  const int q = (int)(t - lt * probes);
  bool alive = false;
  if (lt < P.local_tiles) {
    const int sub = q == 0 ? 11 : (q == 1 ? 22 : (q == 2 ? 17 : 5));  // pixels (3,1) (6,2) (1,2) (5,0) of the tile
    int i, j;
    if (item_pixel(P, (int)(lt << 5) | sub, i, j)) {
      const GlobalScene sc{P.nodes, P.geom};
      Ray r = primary_ray(P, i, j, 0);
      V3 light = v3(1.0f, 1.0f, 1.0f), colour;
      int depth = 0, segments = 0;
      WorkCounters wc;
      do {
        alive = advance_path<false>(sc, P, r, light, depth, colour, wc);
      } while (alive && ++segments < P.probe_segments);
    }
  }
  if (probes > 1) alive |= __shfl_xor_sync(kFullMask, alive, 1);
  if (probes > 2) alive |= __shfl_xor_sync(kFullMask, alive, 2);
  if (q == 0 && lt < P.local_tiles) {
    const long long chunk = lt >> 6;
    const uint32_t pos = (uint32_t)((chunk * P.chunk_stride_inv) % P.n_chunks) << 6 | (uint32_t)(lt & 63);
    keys[lt] = alive ? pos >> 1 : pos;
    ids[lt] = (int32_t)lt;
  }
}

// The probe of a views launch (ray_b200_render_views_into): tile_probe_kernel with each tile traced by its view's camera,
// the 12 floats of `cams` (RayQuery::cams) at its view.
__global__ void __launch_bounds__(256) tile_probe_views_kernel(const __grid_constant__ RenderParams P, uint32_t *__restrict__ keys,
                                                               int32_t *__restrict__ ids, const float *__restrict__ cams) {
  const int probes = P.probes_per_tile;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long lt = t / probes;
  const int q = (int)(t - lt * probes);
  bool alive = false;
  if (lt < P.local_tiles) {
    const int sub = q == 0 ? 11 : (q == 1 ? 22 : (q == 2 ? 17 : 5));
    int v, i, j;
    if (item_view_pixel(P, (int)(lt << 5) | sub, v, i, j)) {
      const GlobalScene sc{P.nodes, P.geom};
      Ray r = primary_ray<false, true>(P, i, j, 0, cams + 12 * (size_t)v);
      V3 light = v3(1.0f, 1.0f, 1.0f), colour;
      int depth = 0, segments = 0;
      WorkCounters wc;
      do {
        alive = advance_path<false>(sc, P, r, light, depth, colour, wc);
      } while (alive && ++segments < P.probe_segments);
    }
  }
  if (probes > 1) alive |= __shfl_xor_sync(kFullMask, alive, 1);
  if (probes > 2) alive |= __shfl_xor_sync(kFullMask, alive, 2);
  if (q == 0 && lt < P.local_tiles) {
    const long long chunk = lt >> 6;
    const uint32_t pos = (uint32_t)((chunk * P.chunk_stride_inv) % P.n_chunks) << 6 | (uint32_t)(lt & 63);
    keys[lt] = alive ? pos >> 1 : pos;
    ids[lt] = (int32_t)lt;
  }
}

// Learned claim order: the probe replaced by what the previous frame of the same scene measured (the longest path of every
// tile, recorded by finish_path).  Tiles with a long path keep their place in the permuted sequence but move in front of
// all others, so the 50-bounce paths that end a frame are claimed in its first few percent.
__global__ void __launch_bounds__(256) tile_cost_keys_kernel(const __grid_constant__ RenderParams P, const uint32_t *__restrict__ cost,
                                                             const int long_path, uint32_t *__restrict__ keys, int32_t *__restrict__ ids) {
  const long long lt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (lt >= P.local_tiles) return;
  const long long chunk = lt >> 6;
  const uint32_t pos = (uint32_t)((chunk * P.chunk_stride_inv) % P.n_chunks) << 6 | (uint32_t)(lt & 63);
  // long_path > 0: two classes (>= long_path first); long_path < 0: four classes with thresholds 8x / 3x / 1x |long_path|
  const uint32_t c = cost[lt];
  uint32_t cls;
  if (long_path > 0) cls = c >= (uint32_t)long_path ? 0u : 3u;
  else { const uint32_t lp = (uint32_t)(-long_path); cls = c >= 8u * lp ? 0u : (c >= 3u * lp ? 1u : (c >= lp ? 2u : 3u)); }
  keys[lt] = (cls << 29) | pos;
  ids[lt] = (int32_t)lt;
}

// ====================================================================================== K3: warp work-queue
// Dense traversal.  K1/K2 bind a lane to a ray for a whole segment, so a warp's SIMT efficiency is
// mean/max of its lanes' traversal lengths.  The reference's
// fold is order-free and never prunes by the running closest t, so a segment's traversal is just a
// SET of independent (ray, node) box-test items and (ray, leaf) sphere-test items.  K3 therefore
// binds lanes to ITEMS, not rays: every warp keeps R = 32*K rays in flight, their traversal items on
// a warp-private queue in shared memory, and each iteration takes 32 items — whatever rays they belong
// to — so every lane does one node step (two box tests) or one sphere test.  Children are pushed back
// with ballot/popc compaction; a sphere hit is folded into its ray's (t, leaf index) pair with two
// 32-bit shared-memory atomicMin (fold_hit), which is exactly the reference's "smallest t, lowest leaf
// index on ties".  When the queues run dry every ray of the round has its closest hit; the owner lanes
// shade, bounce, and idle slots are refilled, and the next round starts.
//
// Queue order and bound.  The order of the items is free, so it serves the batches (see drain): the
// node queue is a ring, batches take its OLDEST items while it is short (breadth-first: only short
// subtrees are left at the end of a round) and the newest above that (depth-first: bounded growth).
// Taken newest-first only, items pushed in reverse lane order keep the queue sorted by tree depth and
// R + 64*(max_depth+1) entries always suffice; the kernel does not rely on that bound: whenever fewer
// than 96 entries are free it takes items one at a time (a plain DFS adds at most `depth` < 64 entries
// before it shrinks), so any ring of >= 256 entries is safe for any content.  Leaf items are drained
// whenever 32 are available, so that stack never holds more than 31 + 64.
//
// Work distribution.  spp == 1 (kSpread = false): a slot owns a pixel (and, for robustness, all its
// samples), claimed from the global cursor with one warp-aggregated atomicAdd.  spp > 1 (kSpread):
// a warp opens up to kRing pixels at a time and hands their samples, in order, to whichever slots are
// idle — consecutive lanes trace consecutive samples of the same pixel (coherent), the scheduling
// grain is one sample instead of one pixel x spp (no long tails, scales to many GPUs), and every
// finished sample's colour is parked in an L2-resident buffer so that the pixel is summed in SAMPLE
// ORDER when its last sample lands, which keeps the result bit-identical to the sequential definition.
//
// The query kind (kQuery, render_params.h Query) says what is traced.  Query::kPixels: camera rays of a frame, as above;
// Q is unused.  Every other kind is a ray query (include/ray_b200.h "ray queries"), "ray mode" below: the work items are
// the caller's rays instead of pixels.  A claim c is ray c (no tile order), a slot is filled from Q.rays, and boxes are
// tested against the query's (t_min, t_max) instead of the literal (0, 1e9).  Rays of a batch are not coherent: ray mode
// has no packet walk and no spread samples.
//
// Query::kClosest, a path or hit query: the closest-hit fold of a frame, spheres tested with epsilon 0.1 whatever t_min
// is (ray.fut:79), the depth limit is Q.max_depth, and a finished path writes Q.rgb / Q.segments.  A hit query
// (Q.hits != NULL, warp-uniform) is a path query of one segment whose owner lane writes the hit record instead of shading.
//
// Query::kAnyHit, an occlusion query: one segment whose answer is "does some leaf the boxes admit accept its sphere in
// (t_min, t_max)", with the query's own t_min (no epsilon).  That is an OR over the set of reached leaves, so it is
// order-free like the closest-hit fold, and it may stop early.  best_t[slot] is a "found" flag (kItemNoHit = nothing yet)
// set by a plain shared store: every writer stores the same value.  Once a slot is marked, its leaf items skip the sphere
// test and its node items push no children, which prunes the rest of that ray's tree; items already queued cost one pop
// each.  The drain still runs the queues dry before a slot is refilled, so no stale item reaches a reused slot, and
// skipping only removes pushes, so the queue bounds and the overflow guard hold as they are.  The owner lane writes
// Q.occluded and frees the slot.  Queue discipline of this kind: node batches as for the other kinds, leaf batches from
// kAnyHitLeafMin items on.
//
// Query::kMultiHit, a multi-hit query: one segment whose answer is every leaf the boxes admit whose sphere accepts in
// (t_min, t_max), again with no epsilon, as the keys bits(t) << 32 | leaf (t >= 0, so bit order is numeric order), of
// which the Q.k smallest are kept and all are counted.  The set of reached leaves does not depend on the order of the
// items, and neither do its k smallest keys nor its size.  The list lives in the ray's own k output records (words 0 and
// 1 of record j = the j-th smallest key so far, sorted); best_t[slot] counts the accepted leaves.  A hit moves the larger
// keys up one record and drops the k-th when the list is full, so a key above the k-th costs one compare.  Lanes of a leaf
// batch that hit the same slot insert one at a time (one lane per slot per round, __syncwarp between rounds); slots are
// warp-private and a ray is claimed once, so no other warp touches the list.  Node batches are those of the closest-hit
// kinds: no box is pruned by the k-th t, because the count needs the whole set.  The owner lane turns the keys into hit
// records (sphere through Q.perm), fills the rest with empty records, writes Q.counts and frees the slot.
//
// kRanged (ray mode, hit / occlusion / multi-hit queries): every ray carries its own interval.  Q.rays is [n][8]
// (struct ray_b200_ray: origin, t_min, direction, t_max), and the per-slot interval takes the place of the query's
// (t_min, t_max) in the root test, the node batch, the leaf batch and the closest-hit finish.  An invalid interval (t_min
// not finite and >= 0, or t_max not finite) becomes (0, 0), which no box passes (tmin >= 0 >= tmax), so the root-miss
// exits write the empty answer.  No shared memory is added: the interval takes the .w words of the slot's float4s that
// the node batch loads anyway, ray_o.w = t_min and ray_i.w = t_max, and a = dot(d, d), which box tests do not use, moves
// to ray_d.w (the leaf batch loads ray_d).  Ranged variants exist only as a separate template instantiation, so the
// per-call variants keep their code.
//
// kAccum (pixel mode, progressive rendering, include/ray_b200.h ray_b200_render_accumulate): the launch traces samples
// [Q.s_begin, Q.s_begin + P.spp) of every pixel.  Everything that counts samples is chunk-relative: P.spp is the chunk
// length (it sizes cbuf and bounds p_ms's 16-bit sample, as spp does for a whole frame), P.offsets starts at the
// chunk's first sample and is read for every sample (primary_ray<true>), and sample rel of the chunk is sample
// s_begin + rel of the frame.  Q.accum holds each pixel's f32 sum of samples [0, s_begin): with s_begin > 0 the in-order
// sum starts from it (p_sum at the pixel-bound refill, the first term of finalize_pixels), with s_begin == 0 from sample
// 0's colour itself, as in a whole frame.  Where the pixel is written (scaled by P.inv_spp = 1/s_end,
// write_pixel<true>), its owner stores the new sum back to Q.accum in place.  So a chain of chunks computes the same f32
// additions in the same order as one frame of s_end samples.
//
// kViews (pixel mode, include/ray_b200.h ray_b200_render_views_into): the launch renders Q.n_views frames of one size
// from one prepared scene.  The work items are the tiles of all views, view after view (P.n_tiles = P.local_tiles =
// n_views * Q.view_tiles), so the chunk permutation of the claim order mixes the views' sky and ground tiles as it mixes
// one frame's.  Where a pixel item becomes a pixel (pixel_of: the pixel-bound refill, finish_path's next sample and store,
// the spread dispenser and finalize_pixels) it also gives its view v; the camera ray reads view v's 12 floats of Q.cams
// instead of P.cam, and the pixel is stored at offset v * H * W.  Nothing else depends on the view, so every view's
// pixel sees exactly the arithmetic of a one-view frame whose P.cam is that camera.

// Query::kAnyHit: a leaf batch runs as soon as this many leaf items are queued (the other kinds wait for 32, a full
// batch), so a ray's first accepted sphere, which ends its traversal, is found sooner.  16 was measured against 1, 8 and
// 32, and newest-first node batches (wq_low = -1) against the default, in DESIGN.md §5.
#ifndef RAYB200_ANYHIT_LEAF_MIN
#define RAYB200_ANYHIT_LEAF_MIN 16
#endif
constexpr int kAnyHitLeafMin = RAYB200_ANYHIT_LEAF_MIN;
static_assert(kAnyHitLeafMin >= 1 && kAnyHitLeafMin <= 32, "a leaf batch takes 1 to 32 items");

template <int K, bool kSpread, bool kPacket, bool kAllNodes, bool kSpheres, Query kQuery = Query::kPixels, bool kRanged = false,
          bool kAccum = false, bool kViews = false>
__global__ void __launch_bounds__(kWqMaxThreads, 1) render_warpqueue_kernel(const __grid_constant__ RenderParams P, const int ncap_arg,
                                                                   const int packet_min, const int refill_min, const int nlow,
                                                                   const __grid_constant__ RayQuery Q) {
  constexpr bool kRays = kQuery != Query::kPixels;  // ray mode
  static_assert(!kRays || (!kSpread && !kPacket), "ray mode traces one ray per slot without spread samples or the packet walk");
  static_assert(!kRanged || kRays, "per-ray intervals belong to ray queries");
  static_assert(!kAccum || !kRays, "progressive rendering accumulates the samples of pixels");
  static_assert(!kViews || (!kRays && !kAccum), "views are whole pixel frames");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  if (P.warp_trace && threadIdx.x == 0) atomicMin(P.warp_trace, global_timer_ns());
  const float4 *s_nodes, *s_geom;
  stage_scene(P, smem_raw, s_nodes, s_geom);
  const StagedScene<kAllNodes, kSpheres> sc{P.nodes, P.geom, s_nodes, s_geom, P.smem_nodes};

  constexpr int R = 32 * K;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the node queue is a ring of the largest power of two that fits its allocation (the launcher hands out powers of two
  // unless a caller asked for an odd capacity)
  const int ncap = 1 << (31 - __clz(ncap_arg));
  const unsigned nmask = (unsigned)ncap - 1u;
  // Oldest-first node batches (see drain) need the ring; they pay everywhere except where the packet walk meets spread
  // samples (64 consecutive samples of a pixel in a warp are coherent already, and the ring costs 8 more instructions per
  // batch), so that combination keeps the plain stack: no index masks, newest first.
  constexpr bool kDeque = !(kPacket && kSpread);
  auto ring = [&](const int i) { return kDeque ? (int)((unsigned)i & nmask) : i; };
  // Lane masks.  At 64 registers the compiler does not keep them live across the batch bodies; re-reading %lanemask_lt/gt
  // is one instruction where re-deriving them from the thread index is four, but it also changes the register
  // allocation: the special registers are used on the packet variants, where that trade paid, and not on the others.
  unsigned lt_mask, gt_mask;
  if constexpr (kPacket) {
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt_mask));
    asm("mov.u32 %0, %%lanemask_gt;" : "=r"(gt_mask));
  } else {
    lt_mask = (1u << lane) - 1u;
    gt_mask = lane == 31 ? 0u : ~((2u << lane) - 1u);
  }
  unsigned char *wbase = smem_raw + ((staging_bytes(P) + 127) & ~(size_t)127) + (size_t)warp * wq_warp_bytes(K, ncap_arg, kPacket, kSpread);
  float4 *ray_o = reinterpret_cast<float4 *>(wbase);   // {o.xyz, a = dot d d}     kRanged: {o.xyz, t_min}
  float4 *ray_i = ray_o + R;                           // {1/d.xyz, 0}             kRanged: {1/d.xyz, t_max}
  float4 *ray_d = ray_i + R;                           // {d.xyz, 0}               kRanged: {d.xyz, a} (t_max until the root test)
  float4 *p_light = ray_d + R;                         // {light.rgb, bits(depth)}   owner lane only
  float4 *p_sum = p_light + R;                         // pixel-bound samples: {sum.rgb, bits(sample)}
  int *p_ms = reinterpret_cast<int *>(p_light + R);    // spread samples: ring entry << 16 | sample (4 bytes per slot instead of 16)
  uint32_t *best_t = kSpread ? reinterpret_cast<uint32_t *>(p_ms + R)   // bits(t) of the closest accepted hit (kItemNoHit = none) ...
                             : reinterpret_cast<uint32_t *>(p_sum + R);
  uint32_t *best_l = best_t + R;                       // ... and its leaf, lowest index among equal t (fold_hit)
  int *p_item = reinterpret_cast<int *>(best_l + R);   // work item (pixel) of the slot, -1 = idle
  int *ring_item = p_item + R;                         // spread: pixel item of ring entry m
  int *ring_done = ring_item + kWqRing;                // spread: samples finished, -1 = entry free
  int *pk_node = ring_done + kWqRing;                  // packet walk: deferred (node, lane mask) pairs, warp-uniform
  unsigned *pk_mask = reinterpret_cast<unsigned *>(pk_node + kWqPacketStack);
  uint32_t *lstk = reinterpret_cast<uint32_t *>(kPacket ? pk_mask + kWqPacketStack : reinterpret_cast<unsigned *>(pk_node));
  uint32_t *nstk = lstk + kWqLeafStack;

  const int total = kRays ? Q.n : (int)(P.local_tiles * kTilePixels);
  const int total_claims = kRays ? Q.n : P.n_chunks << 11;
  // the query's interval (ray mode; kRanged: each slot's own instead) or the literal one of ray_colour (ray.fut:130)
  const float t_lo = kRays ? Q.t_min : 0.0f, t_hi = kRays ? Q.t_max : 1000000000.0f;
  const int spp = P.spp;
#pragma unroll
  for (int k = 0; k < K; k++) p_item[lane + 32 * k] = -1;
  if (lane < kWqRing) ring_done[lane] = -1;
  __syncwarp();
  bool exhausted = false;
  int ntop = 0, nhead = 0, ltop = 0;           // warp-uniform: node queue [nhead, ntop) (ring; nhead = 0 outside drain), leaf stack height
  int open_seq = 0, disp_seq = 0, disp_s = 0;  // spread dispenser (warp-uniform): pixels opened / next sample to hand out
  float4 *cbuf = nullptr;                      // spread: [kWqRing][spp] finished-sample colours of this warp
  if (kSpread) cbuf = P.sample_buf + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * kWqRing * (size_t)spp;
  // kAccum: the running sum of pixel (row pj, column pi), row-major as the frame (64-bit offsets: 2^30 pixels pass 4 GiB)
  [[maybe_unused]] auto accum_of = [&](const int pi, const int pj) { return Q.accum + 3 * ((size_t)pj * P.W + pi); };
  // pixel item -> (view, column, row), false for a padding pixel; the view is 0 unless kViews
  auto pixel_of = [&](const int item, int &pv, int &pi, int &pj) {
    if constexpr (kViews) return item_view_pixel(P, item, pv, pi, pj);
    pv = 0;
    return item_pixel(P, item, pi, pj);
  };
  // kViews: the camera of view pv (its 12 floats of Q.cams)
  [[maybe_unused]] auto view_cam = [&](const int pv) -> const float * { return kViews ? Q.cams + 12 * (size_t)pv : nullptr; };

  // A path in `slot` has ended with `colour`.
  auto finish_path = [&](const int slot, const V3 colour, const int segs) {
    if constexpr (kRays) {
      // a path ended by the depth limit has segs = max_depth + 1 here, but made max_depth objs_hit calls (ray.fut:129)
      const int item = p_item[slot];
      float *c = Q.rgb + 3 * (size_t)item;
      c[0] = colour.x; c[1] = colour.y; c[2] = colour.z;
      if (Q.segments) Q.segments[item] = segs < Q.max_depth ? segs : Q.max_depth;
      p_item[slot] = -1;
      return;
    }
    // learned claim order (recording frame only): the longest path of the tile, sample 0 of its 32 pixels is evidence enough
    if (P.tile_cost && ((kSpread ? p_ms[slot] : __float_as_int(p_sum[slot].w)) & 0xffff) == 0)
      atomicMax(P.tile_cost + (p_item[slot] >> 5), (unsigned)segs);
    if (kSpread) {
      const int ms = p_ms[slot];
      __stcg(cbuf + (size_t)(ms >> 16) * spp + (ms & 0xffff), make_float4(colour.x, colour.y, colour.z, 0.0f));
      atomicAdd(ring_done + (ms >> 16), 1);
      p_item[slot] = -1;
    } else {
      const int item = p_item[slot];
      const float4 ps = p_sum[slot];
      int s = __float_as_int(ps.w);
      // (kAccum: s counts the chunk's samples; only sample 0 of the frame starts the sum, later chunks start from accum)
      const V3 sum = (s == 0 && (!kAccum || Q.s_begin == 0)) ? colour : vadd(v3(ps.x, ps.y, ps.z), colour);
      s++;
      int pi, pj, pv;
      pixel_of(item, pv, pi, pj);
      if (s < spp) {
        const Ray nr = primary_ray<kAccum, kViews>(P, pi, pj, s, view_cam(pv));
        ray_o[slot] = make_float4(nr.o.x, nr.o.y, nr.o.z, 0.0f);
        ray_d[slot] = make_float4(nr.d.x, nr.d.y, nr.d.z, 0.0f);
        p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
        p_sum[slot] = make_float4(sum.x, sum.y, sum.z, __int_as_float(s));
      } else {
        write_pixel<kAccum, kViews>(P, item, pi, pj, sum, pv);
        if constexpr (kAccum) {
          float *a = accum_of(pi, pj);
          a[0] = sum.x; a[1] = sum.y; a[2] = sum.z;
        }
        p_item[slot] = -1;
      }
    }
  };
  // hit query: struct ray_b200_hit of the slot's ray (t = -1, sphere = -1, p = normal = 0 when there is no hit)
  [[maybe_unused]] auto finish_hit = [&](const int slot, const float t, const int sphere, const V3 p, const V3 n) {
    float *h = Q.hits + 8 * (size_t)p_item[slot];
    h[0] = t; h[1] = __int_as_float(sphere);
    h[2] = p.x; h[3] = p.y; h[4] = p.z;
    h[5] = n.x; h[6] = n.y; h[7] = n.z;
    p_item[slot] = -1;
  };
  // multi-hit query: the ray's Q.k records (64-bit offsets: n * k records pass 4 GiB)
  [[maybe_unused]] auto multi_records = [&](const int slot) {
    return reinterpret_cast<uint32_t *>(Q.hits) + (size_t)p_item[slot] * (size_t)Q.k * 8;
  };
  // multi-hit query, one lane per slot at a time: inserts the key (tb, li) into the slot's sorted list of its smallest
  // keys and counts it.  Keys are unique (a ray reaches a leaf once), so the comparisons are strict.
  [[maybe_unused]] auto insert_hit = [&](const int slot, const uint32_t tb, const uint32_t li) {
    const int k = Q.k;
    const uint32_t c = best_t[slot];
    best_t[slot] = c + 1u;
    uint32_t *h = multi_records(slot);
    int j = c < (uint32_t)k ? (int)c : k;  // the key goes to record j, once every larger key has moved up
    for (; j > 0; j--) {
      const uint32_t pt = h[8 * (j - 1)], pl = h[8 * (j - 1) + 1];
      if (pt < tb || (pt == tb && pl < li)) break;
      if (j < k) { h[8 * j] = pt; h[8 * j + 1] = pl; }
    }
    if (j < k) { h[8 * j] = tb; h[8 * j + 1] = li; }
  };
  // multi-hit query, owner lane: the first min(count, k) records hold the sorted keys; each becomes struct ray_b200_hit as
  // the hit query's finish makes it (t, perm[leaf], point_at_param, normal), the rest are empty (t = -1, sphere = -1,
  // p = normal = 0), and the count is the full number of accepted leaves
  [[maybe_unused]] auto finish_multi = [&](const int slot, const uint32_t count) {
    const int k = Q.k;
    uint32_t *h = multi_records(slot);
    const int m = count < (uint32_t)k ? (int)count : k;
    const float4 ro = ray_o[slot], rd = ray_d[slot];
    const V3 o = v3(ro.x, ro.y, ro.z), d = v3(rd.x, rd.y, rd.z);
    // records are 32 bytes: a 16-byte aligned buffer (torch's are) takes two 16-byte stores per record instead of eight
    // scattered 4-byte ones, which was most of the cost of the mostly empty records of large k
    const bool aligned16 = (reinterpret_cast<uintptr_t>(Q.hits) & 15u) == 0;
    for (int j = 0; j < k; j++) {
      float t = -1.0f;
      int sphere = -1;
      V3 p = v3(0.0f, 0.0f, 0.0f), n = p;
      if (j < m) {
        const uint32_t leaf = h[8 * j + 1];
        const float4 g = sc.sphere((int)leaf);
        t = __uint_as_float(h[8 * j]);
        sphere = __ldg(Q.perm + leaf);
        p = vadd(o, vscale(t, d));                                // point_at_param, ray.fut:14-15
        n = vscale(1.0f / g.w, vsub(p, v3(g.x, g.y, g.z)));       // ray.fut:42-43
      }
      if (aligned16) {
        float4 *r = reinterpret_cast<float4 *>(h + 8 * j);
        r[0] = make_float4(t, __int_as_float(sphere), p.x, p.y);
        r[1] = make_float4(p.z, n.x, n.y, n.z);
      } else {
        float *r = reinterpret_cast<float *>(h + 8 * j);
        r[0] = t; r[1] = __int_as_float(sphere);
        r[2] = p.x; r[3] = p.y; r[4] = p.z;
        r[5] = n.x; r[6] = n.y; r[7] = n.z;
      }
    }
    if (Q.counts) Q.counts[p_item[slot]] = (int32_t)count;
    p_item[slot] = -1;
  };
  // spread: pixels whose last sample has landed are summed IN SAMPLE ORDER and written; frees the ring entry
  auto finalize_pixels = [&]() {
    __syncwarp();
    // four lanes per ring entry, one per colour channel: the in-order sum is a dependent chain of spp - 1 additions per
    // channel, so the three channels run side by side instead of one lane doing all three
    const int m = lane >> 2, ch = lane & 3;
    const bool ready = ring_done[m] == spp;
    if (__any_sync(kFullMask, ready)) {
      float sum = 0.0f;
      if (ready && ch < 3) {
        const float *c = reinterpret_cast<const float *>(cbuf + (size_t)m * spp) + ch;
        if constexpr (kAccum) {
          // a later chunk adds its samples to the running sum of the earlier ones, the first chunk starts at its sample 0
          int s = 1, pi, pj;
          if (Q.s_begin > 0 && item_pixel(P, ring_item[m], pi, pj)) {
            sum = accum_of(pi, pj)[ch];
            s = 0;
          } else {
            sum = __ldcg(c);
          }
#pragma unroll 4
          for (; s < spp; s++) sum = sum + __ldcg(c + 4 * s);
        } else {
          sum = __ldcg(c);
#pragma unroll 4
          for (int s = 1; s < spp; s++) sum = sum + __ldcg(c + 4 * s);
        }
      }
      const float g = __shfl_down_sync(kFullMask, sum, 1), b = __shfl_down_sync(kFullMask, sum, 2);
      if (ready && ch == 0) {
        const int item = ring_item[m];
        int pi, pj, pv;
        if (pixel_of(item, pv, pi, pj)) {
          write_pixel<kAccum, kViews>(P, item, pi, pj, v3(sum, g, b), pv);
          if constexpr (kAccum) {
            float *a = accum_of(pi, pj);
            a[0] = sum; a[1] = g; a[2] = b;
          }
        } else if (P.tile_major) {
          P.out_pix[item] = 0;
        }
      }
      __syncwarp();  // every lane of the entry has read ring_done before it is reset
      if (ready && ch == 0) ring_done[m] = -1;
    }
    __syncwarp();
  };

  for (;;) {
    unsigned trav = 0;  // bit k: slot lane+32k has a traversal in flight this round
    // warp-uniform: lanes whose slot lane+32k starts a traversal this round.  (The per-k loops below are NOT unrolled:
    // unrolled, refill / set-up / shading are in the K = 2 kernel twice and its hot code outgrows the SM's instruction cache.)
    unsigned gomask0 = 0u, gomask1 = 0u;
    for (int pass = 0; pass < 4; pass++) {
      // ---------------------------------------------------------------- hand work to idle slots
      if (kSpread) finalize_pixels();
      int my_idle = 0;
#pragma unroll
      for (int k = 0; k < K; k++) my_idle += p_item[lane + 32 * k] < 0;
      int incl = my_idle;  // inclusive warp scan of the idle counts
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(kFullMask, incl, o);
        if (lane >= o) incl += v;
      }
      const int cnt = __shfl_sync(kFullMask, incl, 31);
      int rank = incl - my_idle;
      if (!kSpread) {
        if (cnt && !exhausted) {
          int base = 0;
          if (lane == 0) base = atomicAdd(P.work_cursor, cnt);
          base = __shfl_sync(kFullMask, base, 0);
#pragma unroll 1
          for (int k = 0; k < K; k++) {
            const int slot = lane + 32 * k;
            if (p_item[slot] < 0) {
              const int c = base + rank++;
              const int item = c < total_claims ? (kRays ? c : claim_to_item(P, c)) : total;
              int pi, pj, pv;
              if (kRanged && item < total) {
                // struct ray_b200_ray (64-bit offset: n reaches 2^30); a 16-byte aligned buffer takes two 16-byte loads
                const float *rp = Q.rays + 8 * (size_t)item;
                float4 a, b;
                if ((reinterpret_cast<uintptr_t>(Q.rays) & 15u) == 0) {
                  a = reinterpret_cast<const float4 *>(rp)[0];
                  b = reinterpret_cast<const float4 *>(rp)[1];
                } else {
                  a = make_float4(rp[0], rp[1], rp[2], rp[3]);
                  b = make_float4(rp[4], rp[5], rp[6], rp[7]);
                }
                // the empty answer for an interval the per-call entry points reject: (0, 0) passes no box
                const bool valid = isfinite(a.w) && a.w >= 0.0f && isfinite(b.w);
                p_item[slot] = item;
                ray_o[slot] = make_float4(a.x, a.y, a.z, valid ? a.w : 0.0f);
                ray_d[slot] = make_float4(b.x, b.y, b.z, valid ? b.w : 0.0f);
              } else if (kRays && item < total) {
                const float *rp = Q.rays + 6 * (size_t)item;
                p_item[slot] = item;
                ray_o[slot] = make_float4(rp[0], rp[1], rp[2], 0.0f);
                ray_d[slot] = make_float4(rp[3], rp[4], rp[5], 0.0f);
                p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
              } else if (item < total) {
                if (pixel_of(item, pv, pi, pj)) {
                  const Ray r = primary_ray<kAccum, kViews>(P, pi, pj, 0, view_cam(pv));
                  p_item[slot] = item;
                  ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
                  ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
                  p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
                  if constexpr (kAccum) {  // a later chunk's sum starts from the running sum of the earlier ones
                    float4 ps = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0));
                    if (Q.s_begin > 0) {
                      const float *a = accum_of(pi, pj);
                      ps.x = a[0]; ps.y = a[1]; ps.z = a[2];
                    }
                    p_sum[slot] = ps;
                  } else {
                    p_sum[slot] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0));
                  }
                } else if (P.tile_major) {
                  P.out_pix[item] = 0;
                }
              }
            }
          }
          exhausted = base + cnt >= total_claims;
        }
      } else if (cnt >= refill_min || cnt == R) {
        // (refill_min > 1: wait until several slots are idle, so they get CONSECUTIVE samples and start as a coherent group)
        int avail = (open_seq - disp_seq) * spp - disp_s;
        while (!exhausted && avail < cnt) {  // open more pixels (one cursor claim each) while the ring has room
          const int m = open_seq & (kWqRing - 1);
          if (ring_done[m] != -1) break;
          int c = 0;
          if (lane == 0) c = atomicAdd(P.work_cursor, 1);
          c = __shfl_sync(kFullMask, c, 0);
          if (c >= total_claims) { exhausted = true; break; }
          const int item = claim_to_item(P, c);
          if (item >= total) continue;  // tail of the last (partial) chunk
          __syncwarp();                 // every lane has read ring_done[m] before lane 0 overwrites it
          if (lane == 0) { ring_item[m] = item; ring_done[m] = 0; }
          __syncwarp();
          open_seq++;
          avail += spp;
        }
        const int give = cnt < avail ? cnt : avail;
#pragma unroll 1
        for (int k = 0; k < K; k++) {
          const int slot = lane + 32 * k;
          if (p_item[slot] < 0) {
            const int rk = rank++;
            if (rk < give) {
              int s = disp_s + rk, seq = disp_seq;
              while (s >= spp) { s -= spp; seq++; }
              const int m = seq & (kWqRing - 1);
              const int item = ring_item[m];
              int pi, pj, pv;
              if (pixel_of(item, pv, pi, pj)) {
                const Ray r = primary_ray<kAccum, kViews>(P, pi, pj, s, view_cam(pv));
                p_item[slot] = item;
                ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
                ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
                p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
                p_ms[slot] = (m << 16) | s;
              } else {
                atomicAdd(ring_done + m, 1);  // padding pixel of a partial tile: nothing to trace
              }
            }
          }
        }
        disp_s += give;
        while (disp_s >= spp) { disp_s -= spp; disp_seq++; }
      }
      // -------------------------------------------------------------- set up this round's segments
      // Root box test by the owner lane; a root miss is shaded (sky) on the spot and the path ends,
      // so sky rays never occupy a traversal round.
#pragma unroll 1
      for (int k = 0; k < K; k++) {
        const int slot = lane + 32 * k;
        bool go = false;
        if (!((trav >> k) & 1u)) {
          while (p_item[slot] >= 0) {
            const float4 ro = ray_o[slot], rd = ray_d[slot];
            Ray r;
            r.o = v3(ro.x, ro.y, ro.z);
            r.d = v3(rd.x, rd.y, rd.z);
            const RayInv q = ray_invariants(r);
            const float lo = kRanged ? ro.w : t_lo, hi = kRanged ? rd.w : t_hi;
            if (box_hit(P.root_box[0], P.root_box[1], P.root_box[2], P.root_box[3], P.root_box[4], P.root_box[5], r, q, lo, hi)) {
              if constexpr (kRanged) {
                ray_i[slot] = make_float4(q.ix, q.iy, q.iz, hi);
                ray_d[slot] = make_float4(rd.x, rd.y, rd.z, q.a);
              } else {
                ray_o[slot] = make_float4(ro.x, ro.y, ro.z, q.a);
                ray_i[slot] = make_float4(q.ix, q.iy, q.iz, 0.0f);
              }
              best_t[slot] = kQuery == Query::kMultiHit ? 0u : kItemNoHit;  // multi-hit: no accepted leaf yet
              go = true;
              break;
            }
            // the root box already misses: a one-segment query has its answer
            if constexpr (kQuery == Query::kAnyHit) {  // not occluded
              Q.occluded[p_item[slot]] = 0;
              p_item[slot] = -1;
              continue;
            } else if constexpr (kQuery == Query::kMultiHit) {  // k empty records, count 0
              finish_multi(slot, 0u);
              continue;
            } else if (kQuery == Query::kClosest && (kRanged || Q.hits)) {  // no hit (paths have no ranged form)
              finish_hit(slot, -1.0f, -1, v3(0.0f, 0.0f, 0.0f), v3(0.0f, 0.0f, 0.0f));
              continue;
            }
            const float4 pl = p_light[slot];  // miss (ray.fut:141-148)
            V3 light = v3(pl.x, pl.y, pl.z), colour;
            int depth = __float_as_int(pl.w);
            shade_segment(sc, P, r, q.a, -1, 0.0f, light, depth, colour);
            finish_path(slot, colour, depth + 1);
          }
        }
        const unsigned m = __ballot_sync(kFullMask, go);
        if (go) trav |= 1u << k;
        if (k == 0) gomask0 |= m; else gomask1 |= m;  // the traversal of these rays starts at the root after the passes
      }
      // another pass only helps if some slot is idle and there is still work to hand out
      bool idle_left = false;
#pragma unroll
      for (int k = 0; k < K; k++) idle_left |= p_item[lane + 32 * k] < 0;
      const bool more = kSpread ? (!exhausted || (open_seq - disp_seq) * spp - disp_s > 0) : !exhausted;
      if (!more || !__any_sync(kFullMask, idle_left)) break;
    }
    __syncwarp();
    if ((gomask0 | gomask1) == 0u) {
      bool any_active = false;
#pragma unroll
      for (int k = 0; k < K; k++) any_active |= p_item[lane + 32 * k] >= 0;
      const bool undispensed = kSpread && (open_seq - disp_seq) * spp - disp_s > 0;
      if (exhausted && !undispensed && !__any_sync(kFullMask, any_active)) {
        if (kSpread) finalize_pixels();
        if (P.warp_trace && lane == 0) P.warp_trace[1 + blockIdx.x * (blockDim.x >> 5) + warp] = global_timer_ns();
        break;                                                      // frame done for this warp
      }
      continue;                                                     // only sky / padding so far: hand out more
    }

    // ---------------------------------------------------------------- dense traversal of the round
    // Both batch bodies exist twice: a full-warp version (32 items, no lane predicate: the four push flags stay in
    // predicate registers) used while the queues are deep enough, and a partial one for the drain.
    auto leaf_batch = [&](auto full_tag, const int n_part) {
      // up to 32 (ray, sphere) pairs: closest_hit (ray.fut:78-81) for pixels and closest-hit queries; sphere_hit L[i] r
      // t_min t_max with the query's own t_min (no epsilon) for any-hit and multi-hit queries
      constexpr bool kFull = decltype(full_tag)::value;
      constexpr bool kEpsilon = kQuery == Query::kPixels || kQuery == Query::kClosest;
      const int n = kFull ? 32 : n_part;
      bool hit = false;
      uint32_t tb = 0;
      int slot = 0, li = 0;
      if (kFull || lane < n) {
        const uint32_t it = lstk[ltop - 1 - lane];
        slot = (int)(it >> kSlotShift);
        li = (int)(it & kIndexMask);
        if (kQuery != Query::kAnyHit || best_t[slot] == kItemNoHit) {  // any-hit: items of a marked ray are skipped
          const float4 ro = ray_o[slot], rd = ray_d[slot];
          const float4 g = sc.sphere(li);
          Ray r;
          r.o = v3(ro.x, ro.y, ro.z);
          r.d = v3(rd.x, rd.y, rd.z);
          float a = ro.w, lo = kEpsilon ? 0.1f : t_lo, hi = t_hi;  // epsilon: ray.fut:79
          if constexpr (kRanged) {
            a = rd.w;
            hi = ray_i[slot].w;
            if (!kEpsilon) lo = ro.w;
          }
          const float t = sphere_t(g.x, g.y, g.z, g.w, r, a, lo, hi);
          hit = t >= 0.0f;
          tb = __float_as_uint(t);
        }
      }
      ltop -= n;
      if constexpr (kQuery == Query::kAnyHit) {
        if (hit) best_t[slot] = 0u;  // any value but kItemNoHit: occluded
      } else if constexpr (kQuery == Query::kMultiHit) {
        if (__any_sync(kFullMask, hit)) {
          // every hit into its slot's list: lanes that hit the same slot insert in rounds, the r-th lane of each slot's
          // group in round r
          const unsigned peers = __match_any_sync(kFullMask, hit ? slot : -1);
          const int rank = __popc(peers & lt_mask);
          const int rounds = (int)__reduce_max_sync(kFullMask, hit ? (unsigned)rank + 1u : 0u);
          for (int round = 0; round < rounds; round++) {
            if (hit && rank == round) insert_hit(slot, tb, (uint32_t)li);
            __syncwarp();
          }
        }
      } else {
        fold_hit(best_t, best_l, slot, hit, tb, (uint32_t)li);
      }
    };
    auto node_batch = [&](auto full_tag, const bool bottom, const int n_part) {
      // one BVH2C node step (both children's boxes) for up to 32 (ray, node) pairs, taken from the top of the queue
      // (newest = deepest first) or, `bottom` (warp-uniform), from its bottom (oldest = shallowest first)
      constexpr bool kFull = decltype(full_tag)::value;
      const int n = kFull ? 32 : n_part;
      bool pl_node = false, pr_node = false, pl_leaf = false, pr_leaf = false;
      uint32_t tag = 0;
      int lptr = 0, rptr = 0;
      if (kFull || lane < n) {
        const uint32_t it = nstk[ring(kDeque && bottom ? nhead + lane : ntop + ~lane)];
        tag = it & ~kIndexMask;
        const int slot = (int)(it >> kSlotShift), cur = (int)(it & kIndexMask);
        if (kQuery != Query::kAnyHit || best_t[slot] == kItemNoHit) {  // any-hit: a marked ray pushes nothing, its subtree is pruned
          const float4 ro = ray_o[slot], ri = ray_i[slot];
          float4 q0, q1, q2, q3;
          sc.node(cur, q0, q1, q2, q3);
          Ray r;
          r.o = v3(ro.x, ro.y, ro.z);
          r.d = v3(0.0f, 0.0f, 0.0f);
          RayInv q;
          q.ix = ri.x; q.iy = ri.y; q.iz = ri.z; q.a = ro.w;
          lptr = __float_as_int(q0.w);
          rptr = __float_as_int(q1.w);
          const float lo = kRanged ? ro.w : t_lo, hi = kRanged ? ri.w : t_hi;
          const bool hl = box_hit(q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, r, q, lo, hi);
          const bool hr = box_hit(q2.x, q2.y, q2.z, q3.x, q3.y, q3.z, r, q, lo, hi);
          pl_leaf = lptr < 0;          // a leaf child has no box in the reference: always visited
          pr_leaf = rptr < 0;
          pl_node = hl && !pl_leaf;
          pr_node = hr && !pr_leaf;
        }
      }
      __syncwarp();  // top pops: all of them have been read before anything is pushed over them
      if (kDeque && bottom) nhead += n; else ntop -= n;
      const unsigned bl = __ballot_sync(kFullMask, pl_node), br = __ballot_sync(kFullMask, pr_node);
      // reverse lane order: lane 0 popped the top (deepest) item, its children go back on top
      const int nb = ntop + __popc(bl & gt_mask) + __popc(br & gt_mask);
      if (pr_node) nstk[ring(nb)] = tag | (uint32_t)rptr;
      if (pl_node) nstk[ring(nb + (pr_node ? 1 : 0))] = tag | (uint32_t)lptr;
      ntop += __popc(bl) + __popc(br);
      // two batches in three have no leaf child at all (upper tree levels; the scheduling simulation of rgbbox counts
      // 651 of 973): one vote instead of the two ballots, six popc and the stores
      if (__any_sync(kFullMask, pl_leaf || pr_leaf)) {
        const unsigned cl = __ballot_sync(kFullMask, pl_leaf), cr = __ballot_sync(kFullMask, pr_leaf);
        const int lb = ltop + __popc(cl & lt_mask) + __popc(cr & lt_mask);
        if (pl_leaf) lstk[lb] = tag | (uint32_t)(~lptr);
        if (pr_leaf) lstk[lb + (pl_leaf ? 1 : 0)] = tag | (uint32_t)(~rptr);
        ltop += __popc(cl) + __popc(cr);
      }
    };
    using full_t = std::integral_constant<bool, true>;
    using part_t = std::integral_constant<bool, false>;
    // Runs the item queues dry.  Order is free (the fold is a min), so it is chosen for full batches: while the node
    // queue is short (<= nlow items) batches take its OLDEST items, which widens the frontier breadth-first and leaves only
    // deep items (short subtrees) for the end of the round; above nlow they take the newest (depth-first), which bounds
    // the queue.  With top-only popping the last items of a round are the root-level items at the bottom of the stack,
    // which leaves partial batches at the end of every round; the scheduling simulation of rgbbox rounds (tools/queue_sim.py)
    // gives 0.87 -> 0.98 lane use and 11 % fewer node batches.
    // Overflow guard for ANY content: once fewer than 96 entries are free, items are taken one at a time from the top,
    // a plain DFS that can add at most (tree depth) < 64 entries before it shrinks again.
    auto drain = [&]() {
      __syncwarp();
      const int nroom = ncap - 96;
      constexpr int kLeafMin = kQuery == Query::kAnyHit ? kAnyHitLeafMin : 32;  // leaf items that make a leaf batch due
      for (;;) {
        // the common case first and alone in its loop: full node batches while nothing else is due (the general
        // dispatch below costs ~12 instructions per batch).  One copy of the batch body for both pop directions.
        while ((unsigned)(ntop - nhead - 32) <= (unsigned)(nroom - 32) && ltop < kLeafMin) {
          node_batch(full_t{}, kDeque && ntop - nhead <= nlow, 32);
          __syncwarp();
        }
        const int cnt = ntop - nhead;
        if (ltop >= 32) leaf_batch(full_t{}, 32);
        else if (kLeafMin < 32 && ltop >= kLeafMin) leaf_batch(part_t{}, ltop);
        else if (cnt > 0) node_batch(part_t{}, false, cnt > nroom ? 1 : (cnt < 32 ? cnt : 32));
        else if (ltop > 0) leaf_batch(part_t{}, ltop);
        else break;
        __syncwarp();
      }
      ntop = nhead = 0;  // empty: outside the drain the queue is a plain array again
    };
    // Packet walk.  Near the root almost every ray of a warp visits the same nodes, so those node steps are done the
    // cheap way: ONE (node, lane mask) pair for the whole warp, the node fetched once (same address in every lane =
    // a shared-memory broadcast), each lane testing its own slot's ray, leaf children tested inline by the owner lanes
    // (plain read-modify-write of their own `best` word).  As soon as fewer than `packet_min` lanes are left on a node
    // the remaining (ray, node) pairs are handed to the item queue, where lanes are bound to items instead of rays.
    [[maybe_unused]] auto packet_walk = [&](const int k, unsigned mask) {
      const int slot = lane + 32 * k;
      int cur = 0, psp = 0;
      for (;;) {
        const int cnt = __popc(mask);
        bool descended = false;
        if (cnt < packet_min) {
          if (cnt) {
            if (ntop + 32 + 96 > ncap) drain();
            if ((mask >> lane) & 1u) nstk[ntop + __popc(mask & lt_mask)] = ((uint32_t)slot << kSlotShift) | (uint32_t)cur;
            ntop += cnt;
          }
        } else {
          const bool in = (mask >> lane) & 1u;
          float4 q0, q1, q2, q3;
          sc.node(cur, q0, q1, q2, q3);
          const int lptr = __float_as_int(q0.w), rptr = __float_as_int(q1.w);  // same node in every lane
          bool hl = false, hr = false;
          if (in) {
            const float4 ro = ray_o[slot], ri = ray_i[slot];
            Ray r;
            r.o = v3(ro.x, ro.y, ro.z);
            RayInv q;
            q.ix = ri.x; q.iy = ri.y; q.iz = ri.z; q.a = ro.w;
            r.d = v3(0.0f, 0.0f, 0.0f);
            hl = box_hit(q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, r, q);
            hr = box_hit(q2.x, q2.y, q2.z, q3.x, q3.y, q3.z, r, q);
            if (lptr < 0 || rptr < 0) {  // leaf children: visited by every ray that visits this node (bvh.fut:84)
              const float4 rd = ray_d[slot];
              r.d = v3(rd.x, rd.y, rd.z);
              uint32_t bt = best_t[slot], bl = best_l[slot];  // owner lane, no item of this slot is queued yet: plain update
              if (lptr < 0) {
                const float4 g = sc.sphere(~lptr);
                const float t = sphere_t(g.x, g.y, g.z, g.w, r, ro.w, 0.1f, 1000000000.0f);
                const uint32_t tb = __float_as_uint(t), li = (uint32_t)(~lptr);
                if (t >= 0.0f && (tb < bt || (tb == bt && li < bl))) { bt = tb; bl = li; }
              }
              if (rptr < 0) {
                const float4 g = sc.sphere(~rptr);
                const float t = sphere_t(g.x, g.y, g.z, g.w, r, ro.w, 0.1f, 1000000000.0f);
                const uint32_t tb = __float_as_uint(t), li = (uint32_t)(~rptr);
                if (t >= 0.0f && (tb < bt || (tb == bt && li < bl))) { bt = tb; bl = li; }
              }
              best_t[slot] = bt;
              best_l[slot] = bl;
            }
          }
          const unsigned bl = lptr >= 0 ? __ballot_sync(kFullMask, hl) : 0u;
          const unsigned br = rptr >= 0 ? __ballot_sync(kFullMask, hr) : 0u;
          if (bl) {
            if (br) {
              __syncwarp();  // every lane is done reading the entry this may overwrite
              if (lane == 0) { pk_node[psp] = rptr; pk_mask[psp] = br; }
              psp++;
            }
            cur = lptr; mask = bl; descended = true;
          } else if (br) {
            cur = rptr; mask = br; descended = true;
          }
        }
        if (descended) continue;
        if (psp == 0) break;
        psp--;
        __syncwarp();
        cur = pk_node[psp];
        mask = pk_mask[psp];
      }
    };
#pragma unroll
    for (int k = 0; k < K; k++) {
      const unsigned gm = k == 0 ? gomask0 : gomask1;
      if (kPacket && packet_min > 0) {
        if constexpr (kPacket) {
          if (gm) packet_walk(k, gm);
        }
      } else {
        const bool go = (gm >> lane) & 1u;
        if (go) nstk[ntop + __popc(gm & lt_mask)] = (uint32_t)(lane + 32 * k) << kSlotShift;  // (slot, root node 0)
        ntop += __popc(gm);
      }
    }
    drain();

    // ---------------------------------------------------------------- shade: owner lanes finish the segment
#pragma unroll 1
    for (int k = 0; k < K; k++) {
      if (!((trav >> k) & 1u)) continue;
      const int slot = lane + 32 * k;
      if constexpr (kQuery == Query::kAnyHit) {
        Q.occluded[p_item[slot]] = best_t[slot] != kItemNoHit ? 1 : 0;
        p_item[slot] = -1;
        continue;
      } else if constexpr (kQuery == Query::kMultiHit) {
        finish_multi(slot, best_t[slot]);
        continue;
      }
      const float4 ro = ray_o[slot], rd = ray_d[slot], pl = p_light[slot];
      const uint32_t bt = best_t[slot];
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      V3 light = v3(pl.x, pl.y, pl.z), colour;
      int depth = __float_as_int(pl.w);
      const int j = bt == kItemNoHit ? -1 : (int)best_l[slot];
      const float tb = __uint_as_float(bt);
      if (kQuery == Query::kClosest && (kRanged || Q.hits)) {
        // objs_hit, second half (ray.fut:83-85) with the query's (kRanged: the ray's) t_min; a failed re-intersection is
        // no hit
        float t = -1.0f;
        V3 p = v3(0.0f, 0.0f, 0.0f), n = p;
        if (j >= 0) {
          const float4 g = sc.sphere(j);
          t = kRanged ? sphere_t(g.x, g.y, g.z, g.w, r, rd.w, ro.w, tb + 1.0f)
                      : sphere_t(g.x, g.y, g.z, g.w, r, ro.w, Q.t_min, tb + 1.0f);
          if (t >= 0.0f) {
            p = vadd(r.o, vscale(t, r.d));                            // point_at_param, ray.fut:14-15
            n = vscale(1.0f / g.w, vsub(p, v3(g.x, g.y, g.z)));       // ray.fut:42-43
          }
        }
        if (t >= 0.0f) finish_hit(slot, t, __ldg(Q.perm + j), p, n);
        else finish_hit(slot, -1.0f, -1, p, n);
        continue;
      }
      if (shade_segment(sc, P, r, ro.w, j, tb, light, depth, colour, kRays ? Q.max_depth : kMaxDepth)) {
        ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
        ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
        p_light[slot] = make_float4(light.x, light.y, light.z, __int_as_float(depth));
      } else {
        finish_path(slot, colour, depth + 1);
      }
    }
    __syncwarp();
  }
  signal_frame_done(P);
}

// ====================================================================================== peer-frame flags
// (see include/ray_b200.h "peer-memory frames"): the consumer's stream waits for the producers' kernels through a flag in
// its own memory that the producers bump over NVLink; the producers wait for the consumer's "slot is free again".
__global__ void flag_wait_kernel(const uint32_t *flag, uint32_t value, long long timeout_ns, unsigned long long *timeouts) {
  const unsigned long long t0 = global_timer_ns();
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
    if ((int32_t)(v - value) >= 0) return;
    if (timeout_ns > 0 && (long long)(global_timer_ns() - t0) > timeout_ns) { atomicAdd(timeouts, 1ull); return; }
    __nanosleep(200);
  }
}
__global__ void flag_set_kernel(uint32_t *flag, uint32_t value) {
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}
__global__ void flag_bump_kernel(uint32_t *flag) {
  __threadfence_system();
  atomicAdd_system(flag, 1u);
}

// ====================================================================================== de-tiling (multi-GPU)
// gathered: [world][tiles_padded][32] as an NCCL gather of every rank's compact buffer lays it out.
__global__ void detile_kernel(const int32_t *__restrict__ gathered, int32_t *__restrict__ out, int H, int W, int world,
                              long long tiles_padded, int tiles_x) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)H * W) return;
  const int j = (int)(idx / W), i = (int)(idx - (long long)j * W);
  const long long t = (long long)(j / kTileH) * tiles_x + (i / kTileW);
  const int sub = (j % kTileH) * kTileW + (i % kTileW);
  const long long rank = t % world, lt = t / world;
  out[idx] = gathered[(rank * tiles_padded + lt) * kTilePixels + sub];
}

}  // namespace

// ---------------------------------------------------------------------------------------- host launchers
// Each launcher takes the plan of its frame or query (LaunchConfig: fill_params or the ray-query entry points make it),
// derives the launch geometry once and picks the template instantiation with with_flags (render_common.cuh).  Kernels
// opt in to > 48 KB of dynamic shared memory on first use (launch_opted_in), not at context creation:
// futhark_context_new does not touch the ~50 template instantiations it will never launch.
cudaError_t launch_render(const RenderParams &p, const LaunchConfig &lc, const WavefrontBuffers *wf, cudaStream_t stream,
                          int64_t *launches, const RayQuery *pixq) {
  const long long items = p.local_tiles * kTilePixels;
  if (items <= 0) return cudaSuccess;
  if (lc.kernel == 1) {  // RAY_B200_KERNEL_MEGA
    const int threads = 128;
    const unsigned blocks = (unsigned)((items + threads - 1) / threads);
    render_mega_kernel<false><<<blocks, threads, 0, stream>>>(p);
    (*launches)++;
    return cudaSuccess;
  }
  if (lc.kernel == 6) return launch_lanewalk(p, lc, stream, launches);             // RAY_B200_KERNEL_LANEWALK
  if (lc.kernel != 4) return launch_alt_kernel(p, lc, wf, stream, launches);       // K1 / K2 / K4 (RAYB200_ALL_KERNELS builds)
  return launch_warpqueue(p, Query::kPixels, false, pixq ? *pixq : RayQuery{}, lc, stream, launches);   // RAY_B200_KERNEL_WARPQUEUE
}

// K3: one CTA per SM, wq_warps warps, 32*wq_k rays in flight per warp.  A pixel frame, or a ray query of kind `kind`: the
// same kernel in ray mode, without spread samples or packets; `ranged`: its rays carry their own intervals.
cudaError_t launch_warpqueue(const RenderParams &p, Query kind, bool ranged, const RayQuery &q, const LaunchConfig &lc,
                             cudaStream_t stream, int64_t *launches) {
  const bool rays = kind != Query::kPixels;
  const bool spread = !rays && p.sample_buf != nullptr, packet = !rays && lc.wq_packet > 0;
  const bool accum = !rays && q.accum != nullptr;   // a chunk of a progressive frame
  const bool views = !rays && q.cams != nullptr;    // several views of the scene
  // no more CTAs than there are rays to start at once: a slot takes one query ray, one SAMPLE when samples are spread, one
  // pixel otherwise (capping by pixels alone left 26 SMs idle on a 125 K-pixel shard at 64 spp with 32 warps per CTA)
  const long long work = rays ? (long long)q.n : p.local_tiles * kTilePixels * (spread ? (long long)p.spp : 1ll);
  if (work <= 0) return cudaSuccess;
  const bool all_nodes = p.smem_nodes == p.n_inner, sph = p.smem_spheres == p.n_leaves && p.smem_spheres > 0;
  const int k = lc.wq_k == 1 ? 1 : 2;
  const int wthreads = 32 * lc.wq_warps;
  const int ncap = wq_node_capacity(k, p.max_depth, lc.wq_ncap);
  // breadth-first below this many queued node items (0 = half the ring, < 0 = never: plain LIFO)
  const int nring = 1 << (31 - __builtin_clz((unsigned)ncap));
  const int nlow = lc.wq_low < 0 ? 0 : (lc.wq_low == 0 ? nring / 2 : (lc.wq_low > nring - 96 ? nring - 96 : lc.wq_low));
  const size_t wsmem = ((staging_bytes(p) + 127) & ~(size_t)127) + (size_t)lc.wq_warps * wq_warp_bytes(k, ncap, packet, spread);
  long long ctas = lc.sm_count;
  const long long useful = (work + 32 * k * lc.wq_warps - 1) / (32 * k * lc.wq_warps);
  if (ctas > useful) ctas = useful;
  cudaError_t e;
  if (rays)
    e = with_query([&](auto query) {
      return with_flags([&](auto k2, auto a, auto s, auto rg) {
        return launch_opted_in<render_warpqueue_kernel<k2 ? 2 : 1, false, false, a, s, query, rg>>(
            lc.max_dynamic_smem, (unsigned)ctas, wthreads, wsmem, stream, p, ncap, 0, 1, nlow, q);
      }, k == 2, all_nodes, sph, ranged);
    }, kind);
  else if (views)
    e = with_flags([&](auto k2, auto sp, auto pk, auto a, auto s) {
      return launch_opted_in<render_warpqueue_kernel<k2 ? 2 : 1, sp, pk, a, s, Query::kPixels, false, false, true>>(
          lc.max_dynamic_smem, (unsigned)ctas, wthreads, wsmem, stream, p, ncap, lc.wq_packet, lc.wq_refill, nlow, q);
    }, k == 2, spread, packet, all_nodes, sph);
  else
    e = with_flags([&](auto k2, auto sp, auto pk, auto a, auto s, auto ac) {
      return launch_opted_in<render_warpqueue_kernel<k2 ? 2 : 1, sp, pk, a, s, Query::kPixels, false, ac>>(
          lc.max_dynamic_smem, (unsigned)ctas, wthreads, wsmem, stream, p, ncap, lc.wq_packet, lc.wq_refill, nlow, q);
    }, k == 2, spread, packet, all_nodes, sph, accum);
  if (e == cudaSuccess) (*launches)++;
  return e;
}

// Loads (and opts in to shared memory) the variants the default plan uses - K = 1 / 2, samples spread or not, and the three
// staging cases: whole scene staged, tree partly staged with / without the packet walk - so that the first timed frame of
// main.c does not pay CUDA's lazy function loading.  12 of the 32 pixel instantiations, loaded once per process at
// context creation instead of all kernels of all builds.
cudaError_t preload_default_kernels(int max_dynamic_smem) {
  const bool staging[3][3] = {{false, true, true}, {true, false, false}, {false, false, false}};  // packet, all nodes, spheres
  cudaError_t e = cudaSuccess;
  for (int k2 = 0; k2 < 2; k2++)
    for (int spread = 0; spread < 2; spread++)
      for (const auto &c : staging)
        if (e == cudaSuccess)
          e = with_flags([&](auto kk2, auto sp, auto pk, auto a, auto s) {
            return opt_in_dynamic_smem<render_warpqueue_kernel<kk2 ? 2 : 1, sp, pk, a, s>>(max_dynamic_smem);
          }, k2 == 1, spread == 1, c[0], c[1], c[2]);
  return e;
}

size_t tile_order_sort_bytes(int64_t local_tiles) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                  (int32_t *)nullptr, (int)local_tiles, 0, 32);
  return bytes;
}

void launch_tile_order(const RenderParams &p, const TileOrderBuffers &b, cudaStream_t stream, int64_t *launches,
                       const RayQuery *views) {
  const long long threads = (long long)p.local_tiles * p.probes_per_tile;
  if (views) tile_probe_views_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(p, b.keys, b.ids, views->cams);
  else tile_probe_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(p, b.keys, b.ids);
  size_t bytes = b.sort_tmp_bytes;
  cub::DeviceRadixSort::SortPairs(b.sort_tmp, bytes, b.keys, b.keys_sorted, b.ids, b.order, (int)p.local_tiles, 0,
                                  tile_order_key_bits(p.n_chunks), stream);
  if (launches) *launches += 2;  // the cub sort is counted as one
}

void launch_tile_order_from_cost(const RenderParams &p, const uint32_t *cost, int32_t long_path, const TileOrderBuffers &b,
                                 cudaStream_t stream, int64_t *launches) {
  tile_cost_keys_kernel<<<(unsigned)((p.local_tiles + 255) / 256), 256, 0, stream>>>(p, cost, long_path, b.keys, b.ids);
  size_t bytes = b.sort_tmp_bytes;
  cub::DeviceRadixSort::SortPairs(b.sort_tmp, bytes, b.keys, b.keys_sorted, b.ids, b.order, (int)p.local_tiles, 0, 32, stream);
  if (launches) *launches += 2;
}

void launch_flag_wait(uint32_t *flag, uint32_t value, long long timeout_ns, unsigned long long *timeouts, cudaStream_t stream) {
  flag_wait_kernel<<<1, 1, 0, stream>>>(flag, value, timeout_ns, timeouts);
}
void launch_flag_set(uint32_t *flag, uint32_t value, cudaStream_t stream) { flag_set_kernel<<<1, 1, 0, stream>>>(flag, value); }
void launch_flag_bump(uint32_t *flag, cudaStream_t stream) { flag_bump_kernel<<<1, 1, 0, stream>>>(flag); }

void launch_count_work(const RenderParams &p, cudaStream_t stream, int64_t *launches) {
  const long long items = p.local_tiles * kTilePixels;
  if (items <= 0) return;
  const int threads = 128;
  const unsigned blocks = (unsigned)((items + threads - 1) / threads);
  render_mega_kernel<true><<<blocks, threads, 0, stream>>>(p);
  (*launches)++;
}

void launch_detile(const int32_t *gathered, int32_t *out, int64_t H, int64_t W, int32_t world, int64_t tiles_padded,
                   cudaStream_t stream, int64_t *launches) {
  const long long n = (long long)H * W;
  if (n <= 0) return;
  const int threads = 256;
  const int tiles_x = (int)((W + kTileW - 1) / kTileW);
  detile_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, stream>>>(gathered, out, (int)H, (int)W, world,
                                                                                 tiles_padded, tiles_x);
  (*launches)++;
}

}  // namespace rayb200
