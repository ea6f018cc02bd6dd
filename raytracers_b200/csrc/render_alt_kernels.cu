// The alternative kernels (slower than K3, see DESIGN.md §5), kept with their parity tests: K1
// persistent + lane refill, K2 per-bounce wavefront with global ray queues (the north-star design as specified), K4
// stream queue (K3 without rounds).  Compiled into libray_b200_all.so (-DRAYB200_ALL_KERNELS: the library the test-suite
// loads for these kernels, with K5 from render_lanewalk.cu); the product library libray_b200.so carries only K0 / K3 and
// reports an error for the others, so it stays small and futhark_context_new stays fast.
#include <cub/cub.cuh>
#include "render_common.cuh"

namespace rayb200 {

#ifdef RAYB200_ALL_KERNELS
namespace {

constexpr unsigned long long kNoHit = ~0ull;

// ====================================================================================== K1: persistent + refill
// Persistent CTAs (grid = SMs x resident CTAs).  Every lane owns one pixel at a time and runs its
// samples and bounces; whenever enough lanes of a warp are idle the warp claims new pixels from a
// global cursor with one warp-aggregated atomicAdd (ballot + popc), so irreg's empty-sky rows and
// rgbbox's 50-bounce tails never leave a warp mostly empty.  Samples of one pixel are summed in
// sample order in a register, which is what the spp extension requires.
template <bool kAllNodes, bool kSpheres>
__global__ void __launch_bounds__(256, 2) render_persistent_kernel(const __grid_constant__ RenderParams P,
                                                                    const int refill_min) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const float4 *s_nodes, *s_geom;
  stage_scene(P, smem_raw, s_nodes, s_geom);
  const StagedScene<kAllNodes, kSpheres> sc{P.nodes, P.geom, s_nodes, s_geom, P.smem_nodes};

  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int total = (int)(P.local_tiles * kTilePixels);
  const int total_claims = P.n_chunks << 11;
  WorkCounters wc;

  int item = -1, pi = 0, pj = 0, s = 0, depth = 0;
  Ray r;
  V3 light, sum;
  bool exhausted = false;  // warp-uniform: the cursor has run past the end
  r.o = r.d = light = sum = v3(0.0f, 0.0f, 0.0f);

  for (;;) {
    unsigned idle = __ballot_sync(kFullMask, item < 0);
    if (idle && !exhausted && (__popc(idle) >= refill_min || idle == kFullMask)) {
      const int cnt = __popc(idle);
      const int leader = __ffs(idle) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(P.work_cursor, cnt);
      base = __shfl_sync(kFullMask, base, leader);
      if (item < 0) {
        const int c = base + __popc(idle & lt_mask);
        const int k = c < total_claims ? claim_to_item(P, c) : total;
        if (k < total) {
          if (item_pixel(P, k, pi, pj)) {
            item = k;
            s = 0;
            depth = 0;
            r = primary_ray(P, pi, pj, 0);
            light = v3(1.0f, 1.0f, 1.0f);
          } else if (P.tile_major) {
            P.out_pix[k] = 0;
          }
        }
      }
      exhausted = base + cnt >= total_claims;
      idle = __ballot_sync(kFullMask, item < 0);
    }
    if (idle == kFullMask) {
      if (exhausted) break;
      continue;  // every claimed item was a padding pixel: claim again
    }
    if (item >= 0) {
      V3 colour;
      if (!advance_path<false>(sc, P, r, light, depth, colour, wc)) {
        sum = (s == 0) ? colour : vadd(sum, colour);
        s++;
        if (s < P.spp) {
          depth = 0;
          r = primary_ray(P, pi, pj, s);
          light = v3(1.0f, 1.0f, 1.0f);
        } else {
          write_pixel(P, item, pi, pj, sum);
          item = -1;
        }
      }
    }
  }
}

// ====================================================================================== K2: wavefront
// The north-star design: ONE persistent-threads kernel launch per bounce.  Warps claim batches of 32
// rays from the bounce's global queue with an atomic cursor, trace one segment (same traversal as K1,
// BVH staged by TMA), shade, and append the survivors to the next bounce's queue with warp-vote
// compaction (ballot + popc + one atomicAdd per warp), so every bounce runs on densely packed warps
// whatever the image-space distribution of live paths is.  Bounce 0 generates its rays instead of
// reading them; terminated paths write their pixel (spp == 1) or add into an in-order accumulator.
// From bounce `tail_from` on, the handful of surviving rays are run to completion inside one launch
// instead of paying ~40 more near-empty launches.
template <bool kAllNodes, bool kSpheres>
__global__ void __launch_bounds__(256, 2) wavefront_bounce_kernel(const __grid_constant__ RenderParams P,
                                                                   const __grid_constant__ WavefrontBuffers B,
                                                                   const int bounce, const int sample,
                                                                   const int run_to_end, const int use_order) {
  const long long total64 = P.local_tiles * kTilePixels;
  const int n_in = bounce == 0 ? (int)total64 : B.qlen[bounce];
  if ((long long)blockIdx.x * 32 >= n_in) return;  // nothing for this CTA: skip the staging too
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const float4 *s_nodes, *s_geom;
  stage_scene(P, smem_raw, s_nodes, s_geom);
  const StagedScene<kAllNodes, kSpheres> sc{P.nodes, P.geom, s_nodes, s_geom, P.smem_nodes};
  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int qi = bounce & 1, qo = qi ^ 1;
  const bool last_sample = sample == P.spp - 1;
  WorkCounters wc;
  for (;;) {
    int base = 0;
    if (lane == 0) base = atomicAdd(B.cursor + bounce, 32);
    base = __shfl_sync(kFullMask, base, 0);
    if (base >= n_in) break;
    const int idx = base + lane;
    bool active = idx < n_in;
    Ray r;
    V3 light = v3(1.0f, 1.0f, 1.0f);
    int pid = idx, depth = bounce;
    r.o = r.d = v3(0.0f, 0.0f, 0.0f);
    if (active) {
      if (bounce == 0) {
        int i, j;
        active = item_pixel(P, idx, i, j);
        if (active) r = primary_ray(P, i, j, sample);
        else if (P.tile_major && last_sample) P.out_pix[idx] = 0;
      } else {
        const int src = use_order ? B.order[idx] : idx;  // N4 experiment: trace the queue in (octant, Morton) order
        const float4 a = B.ray_o[qi][src], d = B.ray_d[qi][src], l = B.light[qi][src];
        r.o = v3(a.x, a.y, a.z);
        r.d = v3(d.x, d.y, d.z);
        light = v3(l.x, l.y, l.z);
        depth = __float_as_int(l.w);  // the path state word (render_common.cuh)
        pid = __float_as_int(a.w);
      }
    }
    bool cont = false;
    if (active) {
      V3 colour;
      cont = advance_path<false>(sc, P, r, light, depth, colour, wc);
      if (run_to_end)
        while (cont) cont = advance_path<false>(sc, P, r, light, depth, colour, wc);
      if (!cont) {  // path ended: this sample's colour goes to its pixel, in sample order
        int i, j;
        item_pixel(P, pid, i, j);
        if (P.spp == 1) {
          write_pixel(P, pid, i, j, colour);
        } else {
          V3 sum = colour;
          if (sample > 0) {
            const float4 acc = B.accum[pid];
            sum = vadd(v3(acc.x, acc.y, acc.z), colour);
          }
          if (last_sample) write_pixel(P, pid, i, j, sum);
          else B.accum[pid] = make_float4(sum.x, sum.y, sum.z, 0.0f);
        }
      }
    }
    // warp-vote compaction of the survivors into the next bounce's queue
    const unsigned alive = __ballot_sync(kFullMask, cont);
    if (alive) {
      const int leader = __ffs(alive) - 1;
      int obase = 0;
      if (lane == leader) obase = atomicAdd(B.qlen + bounce + 1, __popc(alive));
      obase = __shfl_sync(kFullMask, obase, leader);
      if (cont) {
        const int o = obase + __popc(alive & lt_mask);
        B.ray_o[qo][o] = make_float4(r.o.x, r.o.y, r.o.z, __int_as_float(pid));
        B.ray_d[qo][o] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
        B.light[qo][o] = make_float4(light.x, light.y, light.z, __int_as_float(depth));
      }
    }
  }
}

// ====================================================================================== K4: stream queue
// K3 without rounds — a NEGATIVE result, kept (like K2) as an alternative with parity tests: it is slower than K3; the
// per-item shared-memory atomics on the ray counters (siblings of one ray sit next to each other in the LIFO, so they
// serialise), the done/free lists and the sparser refill batches cost more than the round tails they remove.
// In K3 a round of 32*K rays cannot end before its slowest ray has walked its ~15 dependent node
// steps, so every round has a tail of partial batches.  K4 keeps the queues permanently
// topped up instead: every ray carries a counter of its outstanding items in shared memory (+children -1 per node item,
// -1 per leaf item); the lane that brings a counter to zero puts the ray on a "done" list; done rays are shaded in dense
// 32-wide batches by whichever lanes are free (all per-ray state lives in shared memory, no owner lanes), and their
// slots — or fresh samples for them — go straight back to the root of the tree while the other rays' items keep the
// node and leaf queues full.  The item LIFO is no longer depth-sorted, so its capacity is protected by the same guard
// as K3's packet spills (one item at a time once fewer than 96 entries are free).
template <int K, bool kSpread, bool kAllNodes, bool kSpheres>
__global__ void __launch_bounds__(kWqMaxThreads, 1) render_streamqueue_kernel(const __grid_constant__ RenderParams P, const int ncap,
                                                                               const int refill_min) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const float4 *s_nodes, *s_geom;
  stage_scene(P, smem_raw, s_nodes, s_geom);
  const StagedScene<kAllNodes, kSpheres> sc{P.nodes, P.geom, s_nodes, s_geom, P.smem_nodes};

  constexpr int R = 32 * K;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  unsigned char *wbase = smem_raw + ((staging_bytes(P) + 127) & ~(size_t)127) + (size_t)warp * sq_warp_bytes(K, ncap);
  float4 *ray_o = reinterpret_cast<float4 *>(wbase);   // {o.xyz, a = dot d d}
  float4 *ray_i = ray_o + R;                           // {1/d.xyz, 0}
  float4 *ray_d = ray_i + R;                           // {d.xyz, 0}
  float4 *p_light = ray_d + R;                         // {light.rgb, bits(depth word, render_common.cuh)}
  float4 *p_sum = p_light + R;                         // {sum.rgb, bits(sample)} / spread: w = bits(ring << 16 | sample)
  unsigned long long *best = reinterpret_cast<unsigned long long *>(p_sum + R);  // (bits(t) << 32 | leaf) min-folded
  int *p_item = reinterpret_cast<int *>(best + R);     // pixel item of the slot, -1 = idle
  int *pending = p_item + R;                           // outstanding traversal items of the slot's ray
  int *ring_item = pending + R;
  int *ring_done = ring_item + kWqRing;
  uint32_t *dstk = reinterpret_cast<uint32_t *>(ring_done + kWqRing);  // slots whose ray has finished its traversal
  uint32_t *fstk = dstk + R;                                           // idle slots
  uint32_t *lstk = fstk + R;
  uint32_t *nstk = lstk + kWqLeafStack;

  const int total = (int)(P.local_tiles * kTilePixels);
  const int total_claims = P.n_chunks << 11;
  const int spp = P.spp;
#pragma unroll
  for (int k = 0; k < K; k++) { p_item[lane + 32 * k] = -1; fstk[lane + 32 * k] = (uint32_t)(lane + 32 * k); }
  if (lane < kWqRing) ring_done[lane] = -1;
  __syncwarp();
  bool exhausted = false;
  int ntop = 0, ltop = 0, dtop = 0, ftop = R;   // warp-uniform stack heights
  int open_seq = 0, disp_seq = 0, disp_s = 0;   // spread dispenser (warp-uniform)
  float4 *cbuf = nullptr;
  if (kSpread) cbuf = P.sample_buf + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * kWqRing * (size_t)spp;

  // A path in `slot` has ended with `colour` (any lane may call this for any slot it is handling).
  auto finish_path = [&](const int slot, const V3 colour) {
    if (kSpread) {
      const int ms = __float_as_int(p_sum[slot].w);
      __stcg(cbuf + (size_t)(ms >> 16) * spp + (ms & 0xffff), make_float4(colour.x, colour.y, colour.z, 0.0f));
      atomicAdd(ring_done + (ms >> 16), 1);
      p_item[slot] = -1;
    } else {
      const int item = p_item[slot];
      const float4 ps = p_sum[slot];
      int s = __float_as_int(ps.w);
      const V3 sum = (s == 0) ? colour : vadd(v3(ps.x, ps.y, ps.z), colour);
      s++;
      int pi, pj;
      item_pixel(P, item, pi, pj);
      if (s < spp) {
        const Ray nr = primary_ray(P, pi, pj, s);
        ray_o[slot] = make_float4(nr.o.x, nr.o.y, nr.o.z, 0.0f);
        ray_d[slot] = make_float4(nr.d.x, nr.d.y, nr.d.z, 0.0f);
        p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
        p_sum[slot] = make_float4(sum.x, sum.y, sum.z, __int_as_float(s));
      } else {
        write_pixel(P, item, pi, pj, sum);
        p_item[slot] = -1;
      }
    }
  };
  auto finalize_pixels = [&]() {
    __syncwarp();
    if (lane < kWqRing && ring_done[lane] == spp) {
      const int item = ring_item[lane];
      int pi, pj;
      if (item_pixel(P, item, pi, pj)) {
        const float4 *c = cbuf + (size_t)lane * spp;
        const float4 c0 = __ldcg(c);
        V3 sum = v3(c0.x, c0.y, c0.z);
        for (int s = 1; s < spp; s++) {
          const float4 cs = __ldcg(c + s);
          sum = vadd(sum, v3(cs.x, cs.y, cs.z));
        }
        write_pixel(P, item, pi, pj, sum);
      } else if (P.tile_major) {
        P.out_pix[item] = 0;
      }
      ring_done[lane] = -1;
    }
    __syncwarp();
  };
  // The slot has a fresh ray (primary or bounced): root box test; sky rays are finished on the spot (which may hand
  // the slot its next sample).  Returns true if the ray enters the tree (its root item is then pushed by the caller).
  auto start_ray = [&](const int slot) -> bool {
    while (p_item[slot] >= 0) {
      const float4 ro = ray_o[slot], rd = ray_d[slot];
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      const RayInv q = ray_invariants(r);
      if (box_hit(P.root_box[0], P.root_box[1], P.root_box[2], P.root_box[3], P.root_box[4], P.root_box[5], r, q)) {
        ray_o[slot] = make_float4(ro.x, ro.y, ro.z, q.a);
        ray_i[slot] = make_float4(q.ix, q.iy, q.iz, 0.0f);
        best[slot] = kNoHit;
        pending[slot] = 1;
        return true;
      }
      const float4 pl = p_light[slot];  // miss (ray.fut:141-148)
      V3 light = v3(pl.x, pl.y, pl.z), colour;
      int depth = __float_as_int(pl.w);
      shade_segment(sc, P, r, q.a, -1, 0.0f, light, depth, colour);
      finish_path(slot, colour);
    }
    return false;
  };
  // After a refill / shade batch: lanes whose ray entered the tree push its root item, lanes whose slot went idle
  // give it back.  `mine`: this lane handled a slot in the batch.
  auto push_roots_and_idle = [&](const bool mine, const int slot, const bool go) {
    const unsigned gm = __ballot_sync(kFullMask, go);
    if (go) nstk[ntop + __popc(gm & lt_mask)] = (uint32_t)slot << kSlotShift;  // (slot, root node 0)
    ntop += __popc(gm);
    const bool idle = mine && !go && p_item[slot] < 0;
    const unsigned im = __ballot_sync(kFullMask, idle);
    if (idle) fstk[ftop + __popc(im & lt_mask)] = (uint32_t)slot;
    ftop += __popc(im);
  };
  auto avail_samples = [&]() { return (open_seq - disp_seq) * spp - disp_s; };

  auto refill = [&]() {
    if (kSpread) finalize_pixels();
    const int f = ftop < 32 ? ftop : 32;
    const bool mine = lane < f;
    const int slot = mine ? (int)fstk[ftop - 1 - lane] : 0;
    __syncwarp();
    ftop -= f;
    if (!kSpread) {
      int base = 0;
      if (lane == 0) base = atomicAdd(P.work_cursor, f);
      base = __shfl_sync(kFullMask, base, 0);
      if (mine) {
        const int c = base + lane;
        const int item = c < total_claims ? claim_to_item(P, c) : total;
        int pi, pj;
        if (item < total) {
          if (item_pixel(P, item, pi, pj)) {
            const Ray r = primary_ray(P, pi, pj, 0);
            p_item[slot] = item;
            ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
            ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
            p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
            p_sum[slot] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0));
          } else if (P.tile_major) {
            P.out_pix[item] = 0;
          }
        }
      }
      exhausted = base + f >= total_claims;
    } else {
      int avail = avail_samples();
      while (!exhausted && avail < f) {  // open more pixels while the ring has room
        const int m = open_seq & (kWqRing - 1);
        if (ring_done[m] != -1) break;
        int c = 0;
        if (lane == 0) c = atomicAdd(P.work_cursor, 1);
        c = __shfl_sync(kFullMask, c, 0);
        if (c >= total_claims) { exhausted = true; break; }
        const int item = claim_to_item(P, c);
        if (item >= total) continue;
        __syncwarp();
        if (lane == 0) { ring_item[m] = item; ring_done[m] = 0; }
        __syncwarp();
        open_seq++;
        avail += spp;
      }
      const int give = f < avail ? f : avail;
      if (mine && lane < give) {
        int s = disp_s + lane, seq = disp_seq;
        while (s >= spp) { s -= spp; seq++; }
        const int m = seq & (kWqRing - 1);
        const int item = ring_item[m];
        int pi, pj;
        if (item_pixel(P, item, pi, pj)) {
          const Ray r = primary_ray(P, pi, pj, s);
          p_item[slot] = item;
          ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
          ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
          p_light[slot] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
          p_sum[slot] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float((m << 16) | s));
        } else {
          atomicAdd(ring_done + m, 1);  // padding pixel of a partial tile: nothing to trace
        }
      }
      disp_s += give;
      while (disp_s >= spp) { disp_s -= spp; disp_seq++; }
    }
    const bool go = mine ? start_ray(slot) : false;
    push_roots_and_idle(mine, slot, go);
  };

  auto shade_batch = [&]() {
    const int d = dtop < 32 ? dtop : 32;
    const bool mine = lane < d;
    const int slot = mine ? (int)dstk[dtop - 1 - lane] : 0;
    __syncwarp();
    dtop -= d;
    bool go = false;
    if (mine) {
      const float4 ro = ray_o[slot], rd = ray_d[slot], pl = p_light[slot];
      const unsigned long long b = best[slot];
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      V3 light = v3(pl.x, pl.y, pl.z), colour;
      int depth = __float_as_int(pl.w);
      const int j = b == kNoHit ? -1 : (int)(unsigned)(b & 0xffffffffu);
      const float tb = __uint_as_float((unsigned)(b >> 32));
      if (shade_segment(sc, P, r, ro.w, j, tb, light, depth, colour)) {
        ray_o[slot] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
        ray_d[slot] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
        p_light[slot] = make_float4(light.x, light.y, light.z, __int_as_float(depth));
      } else {
        finish_path(slot, colour);
      }
      go = start_ray(slot);
    }
    push_roots_and_idle(mine, slot, go);
  };

  auto leaf_batch = [&](auto full_tag) {
    constexpr bool kFull = decltype(full_tag)::value;
    const int n = kFull ? 32 : ltop;
    bool done = false;
    int slot = 0;
    if (kFull || lane < n) {
      const uint32_t it = lstk[ltop - 1 - lane];
      slot = (int)(it >> kSlotShift);
      const int li = (int)(it & kIndexMask);
      const float4 ro = ray_o[slot], rd = ray_d[slot];
      const float4 g = sc.sphere(li);
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      const float t = sphere_t(g.x, g.y, g.z, g.w, r, ro.w, 0.1f, 1000000000.0f);
      if (t >= 0.0f) atomicMin(best + slot, ((unsigned long long)__float_as_uint(t) << 32) | (unsigned)li);
      done = atomicSub(pending + slot, 1) == 1;  // this was the ray's last outstanding item
    }
    ltop -= n;
    const unsigned dm = __ballot_sync(kFullMask, done);
    if (done) dstk[dtop + __popc(dm & lt_mask)] = (uint32_t)slot;
    dtop += __popc(dm);
  };
  auto node_batch = [&](auto full_tag, const int n_part) {
    constexpr bool kFull = decltype(full_tag)::value;
    const int n = kFull ? 32 : n_part;
    bool pl_node = false, pr_node = false, pl_leaf = false, pr_leaf = false, done = false;
    uint32_t tag = 0;
    int lptr = 0, rptr = 0, slot = 0;
    if (kFull || lane < n) {
      const uint32_t it = nstk[ntop - 1 - lane];
      tag = it & ~kIndexMask;
      slot = (int)(it >> kSlotShift);
      const int cur = (int)(it & kIndexMask);
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
      const bool hl = box_hit(q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, r, q);
      const bool hr = box_hit(q2.x, q2.y, q2.z, q3.x, q3.y, q3.z, r, q);
      pl_leaf = lptr < 0;
      pr_leaf = rptr < 0;
      pl_node = hl && !pl_leaf;
      pr_node = hr && !pr_leaf;
      const int delta = (int)pl_node + (int)pr_node + (int)pl_leaf + (int)pr_leaf - 1;
      if (delta != 0) done = atomicAdd(pending + slot, delta) + delta == 0;
    }
    __syncwarp();  // all pops have been read before anything is pushed over them
    ntop -= n;
    const unsigned bl = __ballot_sync(kFullMask, pl_node), br = __ballot_sync(kFullMask, pr_node);
    const unsigned cl = __ballot_sync(kFullMask, pl_leaf), cr = __ballot_sync(kFullMask, pr_leaf);
    const int nb = ntop + __popc(bl & lt_mask) + __popc(br & lt_mask);
    if (pl_node) nstk[nb] = tag | (uint32_t)lptr;
    if (pr_node) nstk[nb + (pl_node ? 1 : 0)] = tag | (uint32_t)rptr;
    ntop += __popc(bl) + __popc(br);
    const int lb = ltop + __popc(cl & lt_mask) + __popc(cr & lt_mask);
    if (pl_leaf) lstk[lb] = tag | (uint32_t)(~lptr);
    if (pr_leaf) lstk[lb + (pl_leaf ? 1 : 0)] = tag | (uint32_t)(~rptr);
    ltop += __popc(cl) + __popc(cr);
    const unsigned dm = __ballot_sync(kFullMask, done);
    if (done) dstk[dtop + __popc(dm & lt_mask)] = (uint32_t)slot;
    dtop += __popc(dm);
  };
  using full_t = std::integral_constant<bool, true>;
  using part_t = std::integral_constant<bool, false>;

  for (;;) {
    const bool work_left = kSpread ? (!exhausted || avail_samples() > 0) : !exhausted;
    // a refill must be able to hand something out, or the loop would spin on it: samples already opened, or a ring entry
    // that is free / can be finalized right now
    bool can_hand_out = work_left;
    if (kSpread && avail_samples() <= 0) {
      const int rd = ring_done[open_seq & (kWqRing - 1)];
      can_hand_out = !exhausted && (rd == -1 || rd == spp);
    }
    const bool can_refill = ftop > 0 && can_hand_out;
    const bool tight = ntop + 96 > ncap;
    if (dtop >= 32) shade_batch();
    else if (ltop >= 32) leaf_batch(full_t{});
    else if (ntop >= 32 && !tight) node_batch(full_t{}, 32);
    else if (can_refill && ftop >= refill_min && !tight) refill();   // top the queues up before running partial batches
    else if (dtop > 0) shade_batch();
    else if (ntop > 0) node_batch(part_t{}, tight ? 1 : (ntop < 32 ? ntop : 32));
    else if (ltop > 0) leaf_batch(part_t{});
    else if (can_refill) refill();
    else if (kSpread && ftop == R && !work_left) {
      // everything handed out and finished: flush the last pixels; if that frees nothing there is nothing left
      finalize_pixels();
      break;
    } else break;
    __syncwarp();
  }
}

// N4 experiment: sort key of queue entry i for `bounce` = direction octant (3 bits) | 29-bit Morton code of the origin
// normalised to the root box; entries past the queue's length sort last.
__device__ __forceinline__ uint32_t spread10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}
__global__ void wavefront_sort_keys_kernel(const __grid_constant__ RenderParams P, const __grid_constant__ WavefrontBuffers B,
                                           const int bounce) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B.capacity) return;
  const int n = B.qlen[bounce], qi = bounce & 1;
  uint32_t key = 0xffffffffu;
  if (i < n) {
    const float4 o = B.ray_o[qi][i], d = B.ray_d[qi][i];
    const float sx = 1023.0f / fmaxf(P.root_box[3] - P.root_box[0], 1e-20f), sy = 1023.0f / fmaxf(P.root_box[4] - P.root_box[1], 1e-20f),
                sz = 1023.0f / fmaxf(P.root_box[5] - P.root_box[2], 1e-20f);
    const uint32_t x = (uint32_t)fminf(fmaxf((o.x - P.root_box[0]) * sx, 0.0f), 1023.0f);
    const uint32_t y = (uint32_t)fminf(fmaxf((o.y - P.root_box[1]) * sy, 0.0f), 1023.0f);
    const uint32_t z = (uint32_t)fminf(fmaxf((o.z - P.root_box[2]) * sz, 0.0f), 1023.0f);
    const uint32_t m = (spread10(x) << 2) | (spread10(y) << 1) | spread10(z);
    const uint32_t oct = (d.x < 0.0f ? 4u : 0u) | (d.y < 0.0f ? 2u : 0u) | (d.z < 0.0f ? 1u : 0u);
    key = (oct << 29) | (m >> 1);
    if (key == 0xffffffffu) key = 0xfffffffeu;
  }
  B.sort_keys[i] = key;
  B.sort_ids[i] = (int32_t)i;
}

}  // namespace

size_t wavefront_sort_bytes(int64_t items) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                  (int32_t *)nullptr, (int)items, 0, 32);
  return bytes;
}

cudaError_t launch_alt_kernel(const RenderParams &p, const LaunchConfig &lc, const WavefrontBuffers *wf, cudaStream_t stream,
                              int64_t *launches) {
  const long long items = p.local_tiles * kTilePixels;
  const int threads = 256;
  const size_t smem = staging_bytes(p);
  const bool all_nodes = p.smem_nodes == p.n_inner, sph = p.smem_spheres == p.n_leaves && p.smem_spheres > 0;
  long long want = (long long)lc.sm_count * lc.blocks_per_sm;
  cudaError_t e = cudaSuccess;
  switch (lc.kernel) {
  case RAY_B200_KERNEL_WAVEFRONT: {  // per sample pass, one launch per bounce up to the tail bounce
    const long long max_useful = (items + 31) / 32;
    if (want > max_useful) want = max_useful;
    const int tail = wf->tail_from < 0 ? 0 : (wf->tail_from > kMaxDepth - 1 ? kMaxDepth - 1 : wf->tail_from);
    for (int s = 0; s < p.spp && e == cudaSuccess; s++) {
      cudaMemsetAsync(wf->qlen, 0, 2 * (kMaxDepth + 2) * sizeof(int32_t), stream);  // qlen and cursor are contiguous
      for (int b = 0; b <= tail && e == cudaSuccess; b++) {
        const int rte = b == tail;
        const int use_order = (b >= 1 && b <= wf->sort_bounces && wf->order != nullptr) ? 1 : 0;
        if (use_order) {  // N4 experiment: order the queue this bounce reads
          wavefront_sort_keys_kernel<<<(unsigned)((wf->capacity + 255) / 256), 256, 0, stream>>>(p, *wf, b);
          size_t tmp = wf->sort_tmp_bytes;
          cub::DeviceRadixSort::SortPairs(wf->sort_tmp, tmp, wf->sort_keys, wf->sort_keys_out, wf->sort_ids, wf->order,
                                          (int)wf->capacity, 0, 32, stream);
          (*launches) += 2;
        }
        e = with_flags([&](auto a, auto spheres) {  // (s is the sample pass)
          return launch_opted_in<wavefront_bounce_kernel<a, spheres>>(lc.max_dynamic_smem, (unsigned)want, threads, smem,
                                                                      stream, p, *wf, b, s, rte, use_order);
        }, all_nodes, sph);
        (*launches)++;
      }
    }
    return e;
  }
  case RAY_B200_KERNEL_STREAMQUEUE: {  // one CTA per SM, rays refilled continuously (no rounds); 32 rays per warp
    constexpr int k = 1;
    const int wthreads = 32 * lc.wq_warps;
    const int ncap = wq_node_capacity(k, p.max_depth);
    const size_t wsmem = ((staging_bytes(p) + 127) & ~(size_t)127) + (size_t)lc.wq_warps * sq_warp_bytes(k, ncap);
    long long ctas = lc.sm_count;
    const bool spread = p.sample_buf != nullptr;
    const long long rays = items * (spread ? (long long)p.spp : 1ll);
    const long long useful = (rays + 32 * k * lc.wq_warps - 1) / (32 * k * lc.wq_warps);
    if (ctas > useful) ctas = useful;
    e = with_flags([&](auto sp, auto a, auto s) {
      return launch_opted_in<render_streamqueue_kernel<k, sp, a, s>>(lc.max_dynamic_smem, (unsigned)ctas, wthreads, wsmem,
                                                                     stream, p, ncap, lc.wq_refill);
    }, spread, all_nodes, sph);
    if (e == cudaSuccess) (*launches)++;
    return e;
  }
  case RAY_B200_KERNEL_PERSISTENT: break;
  default: return cudaErrorInvalidValue;
  }
  const long long max_useful = (items + threads - 1) / threads;
  if (want > max_useful) want = max_useful;
  const int refill = lc.refill_min < 1 ? 1 : (lc.refill_min > 32 ? 32 : lc.refill_min);
  e = with_flags([&](auto a, auto s) {
    return launch_opted_in<render_persistent_kernel<a, s>>(lc.max_dynamic_smem, (unsigned)want, threads, smem, stream, p, refill);
  }, all_nodes, sph);
  if (e == cudaSuccess) (*launches)++;
  return e;
}
#else   // product build: the alternatives are not compiled in

size_t wavefront_sort_bytes(int64_t) { return 0; }

cudaError_t launch_alt_kernel(const RenderParams &, const LaunchConfig &, const WavefrontBuffers *, cudaStream_t, int64_t *) {
  return cudaErrorNotSupported;
}
#endif

}  // namespace rayb200
