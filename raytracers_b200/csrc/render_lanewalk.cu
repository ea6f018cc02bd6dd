// K5 `render_lanewalk_kernel` — lane-owned traversals, slot-owned paths, no rounds (sm_90a).
//
// The reference's hot loop (ray.fut:126-148 over bvh.fut:61-84 / ray.fut:53-70) as K3 runs it costs ~114 warp
// instructions and ~110 B of shared-memory traffic per 32 node steps, of which only 46 instructions and 64 B are the two
// box tests and the node record: the rest re-binds lanes to (ray, node) items every step (pop, ray fetch, two-level
// ballot compaction, push), so issue slots AND the shared-memory pipe are both busy with bookkeeping.  K5 keeps the
// part of K3 that works — paths live in shared-memory SLOTS, not in lanes; sphere tests are (ray, leaf) items drained
// in dense batches; samples of a pixel are spread and summed in sample order — and changes who walks the tree:
//
//   * a LANE owns one ray's whole traversal: origin and 1/direction stay in registers, the DFS stack is a private
//     column of a [depth][32] shared-memory array (bank = lane: conflict-free), the next node comes straight out of the
//     box tests — no item pop, no ray fetch, no compaction on the node path: ~85 instructions and ~72 B per 32 steps;
//   * there are NO rounds: a lane whose traversal ends puts the slot on the warp's `done` list and takes the next slot
//     from the `ready` list in the same iteration, so lanes stay busy while other rays of the warp are still walking;
//     with R > 32 slots per warp the shading of finished segments happens in dense batches (up to 32 slots, any lanes)
//     and refills `ready` before it runs dry;
//   * rays that start together (consecutive samples of one pixel) walk the top of the tree in lockstep, so their node
//     fetches are same-address broadcasts — the packet walk of K3 for free;
//   * a single path's latency is one dependent LDS + box test per level (~100-150 cycles staged) instead of K3's
//     pop -> fetch -> test -> ballot -> push -> sync chain: the 50-bounce paths a frame ends on finish ~3x sooner.
//
// Exactness is unchanged (DESIGN.md §2): the set of leaves visited is order-free, sphere hits are folded per slot as
// "smallest t, lowest leaf index on ties" (fold_hit), shading is K3's shade_segment, samples are summed in sample order.
//
// Not the default (resolve_kernel picks K3): the step itself is the ~85 instructions estimated above, but the
// per-iteration list maintenance (finished lanes -> done list, idle lanes <- ready list: two ballots, popc, byte-list
// traffic, ray reload) costs another ~75 and the leaf-item push ~35, so an iteration is ~200 instructions for 32 steps
// against K3's ~114; and un-staged nodes are fetched per lane without K3's packet sharing.  Kept, like K1 / K2 / K4, as an
// alternative with the same parity tests, in the RAYB200_ALL_KERNELS build only.
#include "render_common.cuh"

namespace rayb200 {

#ifdef RAYB200_ALL_KERNELS
namespace {

constexpr int kLwFin = -1;    // lane state: traversal just ended, the slot is still in `tag`
constexpr int kLwIdle = -2;   // lane state: no slot
constexpr uint32_t kLwNoHit = kItemNoHit;

template <int R, bool kSpread, bool kAllNodes, bool kSpheres>
__global__ void __launch_bounds__(kWqMaxThreads, 1) render_lanewalk_kernel(const __grid_constant__ RenderParams P, const int scap,
                                                                            const int idle_min, const int max_pass) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  if (P.warp_trace && threadIdx.x == 0) atomicMin(P.warp_trace, global_timer_ns());
  const float4 *s_nodes, *s_geom;
  stage_scene(P, smem_raw, s_nodes, s_geom);
  const StagedScene<kAllNodes, kSpheres> sc{P.nodes, P.geom, s_nodes, s_geom, P.smem_nodes};

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  // R is a template parameter so that every per-warp array sits at a compile-time offset from ONE base register (with a
  // runtime slot count the 16 array pointers alone pushed the walking lane's ray into local memory)
  unsigned char *wbase = smem_raw + ((staging_bytes(P) + 127) & ~(size_t)127) + (size_t)warp * lw_warp_bytes(R, scap);
  float4 *ray_o = reinterpret_cast<float4 *>(wbase);   // {o.xyz, a = dot d d}
  float4 *ray_i = ray_o + R;                           // {1/d.xyz, 0}
  float4 *ray_d = ray_i + R;                           // {d.xyz, 0}
  float4 *p_light = ray_d + R;                         // {light.rgb, bits(depth word, render_common.cuh)}
  uint32_t *best_t = reinterpret_cast<uint32_t *>(p_light + R);  // bits(t) of the closest accepted hit, kLwNoHit = none
  uint32_t *best_l = best_t + R;                       // its leaf (lowest index among equal t)
  int *p_item = reinterpret_cast<int *>(best_l + R);   // pixel item of the slot
  int *p_meta = p_item + R;                            // spread: ring entry << 16 | sample
  int *ring_item = p_meta + R;                         // spread: pixel item of ring entry m
  int *ring_done = ring_item + kWqRing;                // spread: samples finished, -1 = entry free
  uint32_t *lstk = reinterpret_cast<uint32_t *>(ring_done + kWqRing);   // (slot, leaf) items awaiting a sphere test
  unsigned char *ready = reinterpret_cast<unsigned char *>(lstk + kWqLeafStack);  // slots whose traversal can start
  unsigned char *done = ready + R;                     // slots whose traversal has ended (awaiting the leaf flush + shading)
  unsigned char *freel = done + R;                     // slots without a path
  uint32_t *stk = reinterpret_cast<uint32_t *>(ready + ((3 * R + 15) & ~15));  // private DFS stacks, [scap][32] (last: scap is a runtime value)

  const int total = (int)(P.local_tiles * kTilePixels);
  const int total_claims = P.n_chunks << 11;
  const int spp = P.spp;
  for (int s = lane; s < R; s += 32) freel[s] = (unsigned char)s;
  if (lane < kWqRing) ring_done[lane] = -1;
  __syncwarp();
  bool exhausted = false;
  int nready = 0, ndone = 0, nfree = R, ltop = 0;   // warp-uniform list heights
  int open_seq = 0, disp_seq = 0, disp_s = 0;       // spread dispenser (warp-uniform): pixels opened / next sample to hand out
  float4 *cbuf = nullptr;                           // spread: [kWqRing][spp] finished-sample colours of this warp
  if (kSpread) cbuf = P.sample_buf + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * kWqRing * (size_t)spp;

  // lane-owned traversal state
  int cur = kLwIdle;
  uint32_t tag = 0;                                  // slot << kSlotShift
  float ox = 0.0f, oy = 0.0f, oz = 0.0f, ix = 0.0f, iy = 0.0f, iz = 0.0f;
  uint32_t *const sbase = stk + lane;
  uint32_t *sp = sbase;

  // A path in `slot` has ended with `colour`.
  auto finish_path = [&](const int slot, const V3 colour) {
    if (kSpread) {
      const int ms = p_meta[slot];
      __stcg(cbuf + (size_t)(ms >> 16) * spp + (ms & 0xffff), make_float4(colour.x, colour.y, colour.z, 0.0f));
      atomicAdd(ring_done + (ms >> 16), 1);
    } else {
      const int item = p_item[slot];
      int pi, pj;
      item_pixel(P, item, pi, pj);
      write_pixel(P, item, pi, pj, colour);
    }
  };
  // spread: pixels whose last sample has landed are summed IN SAMPLE ORDER and written; frees the ring entry
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
  auto undispensed = [&]() { return kSpread ? (open_seq - disp_seq) * spp - disp_s : 0; };

  // closest_hit (ray.fut:78-81) for up to 32 (slot, sphere) items; the hits are folded per slot
  auto leaf_batch = [&](const int n) {
    bool hit = false;
    uint32_t tb = 0;
    int slot = 0, li = 0;
    if (lane < n) {
      const uint32_t it = lstk[ltop - 1 - lane];
      slot = (int)(it >> kSlotShift);
      li = (int)(it & kIndexMask);
      const float4 ro = ray_o[slot], rd = ray_d[slot];
      const float4 g = sc.sphere(li);
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      const float t = sphere_t(g.x, g.y, g.z, g.w, r, ro.w, 0.1f, 1000000000.0f);
      hit = t >= 0.0f;
      tb = __float_as_uint(t);
    }
    ltop -= n;
    fold_hit(best_t, best_l, slot, hit, tb, (uint32_t)li);
  };
  auto drain_leaves = [&]() {
    while (ltop > 0) leaf_batch(ltop < 32 ? ltop : 32);
  };

  // Shading + refill.  Takes up to 32 slots off the done list (their sphere items have been flushed), finishes the
  // segment (ray.fut:130-148), and keeps handing work to slots without a path until the ready list has been topped up:
  // a continued or fresh ray gets its invariants and the root box test here (a root miss is shaded as sky on the spot),
  // so a slot on the ready list always starts its walk at node 0.
  auto shade_phase = [&]() {
    if (kSpread) finalize_pixels();
    const int nb = ndone < 32 ? ndone : 32;
    int my = -1, state = 0;   // 0: no slot, 1: slot with a ray to set up, 2: slot without a path
    if (lane < nb) {
      my = done[ndone - 1 - lane];
      const float4 ro = ray_o[my], rd = ray_d[my], pl = p_light[my];
      const uint32_t bt = best_t[my];
      Ray r;
      r.o = v3(ro.x, ro.y, ro.z);
      r.d = v3(rd.x, rd.y, rd.z);
      V3 light = v3(pl.x, pl.y, pl.z), colour;
      int depth = __float_as_int(pl.w);
      const int j = bt == kLwNoHit ? -1 : (int)best_l[my];
      if (shade_segment(sc, P, r, ro.w, j, __uint_as_float(bt), light, depth, colour)) {
        ray_o[my] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
        ray_d[my] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
        p_light[my] = make_float4(light.x, light.y, light.z, __int_as_float(depth));
        state = 1;
      } else {
        finish_path(my, colour);
        state = 2;
      }
    }
    ndone -= nb;
    for (int pass = 0; pass < max_pass; pass++) {
      // lanes without a slot adopt one from the free list
      const unsigned none = __ballot_sync(kFullMask, state == 0);
      if (none && nfree > 0) {
        const int rk = __popc(none & lt_mask), n = min(__popc(none), nfree);
        if (state == 0 && rk < n) { my = freel[nfree - 1 - rk]; state = 2; }
        nfree -= n;
      }
      // hand new work to the slots without a path
      const unsigned want = __ballot_sync(kFullMask, state == 2);
      const int cnt = __popc(want);
      const int rank = __popc(want & lt_mask);
      if (kSpread) finalize_pixels();
      if (!kSpread) {
        if (cnt && !exhausted) {
          int base = 0;
          if (lane == 0) base = atomicAdd(P.work_cursor, cnt);
          base = __shfl_sync(kFullMask, base, 0);
          if (state == 2) {
            const int c = base + rank;
            const int item = c < total_claims ? claim_to_item(P, c) : total;
            int pi, pj;
            if (item < total) {
              if (item_pixel(P, item, pi, pj)) {
                const Ray r = primary_ray(P, pi, pj, 0);
                p_item[my] = item;
                ray_o[my] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
                ray_d[my] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
                p_light[my] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
                state = 1;
              } else if (P.tile_major) {
                P.out_pix[item] = 0;
              }
            }
          }
          exhausted = base + cnt >= total_claims;
        }
      } else if (cnt) {
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
        if (state == 2 && rank < give) {
          int s = disp_s + rank, seq = disp_seq;
          while (s >= spp) { s -= spp; seq++; }
          const int m = seq & (kWqRing - 1);
          const int item = ring_item[m];
          int pi, pj;
          if (item_pixel(P, item, pi, pj)) {
            const Ray r = primary_ray(P, pi, pj, s);
            p_item[my] = item;
            p_meta[my] = (m << 16) | s;
            ray_o[my] = make_float4(r.o.x, r.o.y, r.o.z, 0.0f);
            ray_d[my] = make_float4(r.d.x, r.d.y, r.d.z, 0.0f);
            p_light[my] = make_float4(1.0f, 1.0f, 1.0f, __int_as_float(0));
            state = 1;
          } else {
            atomicAdd(ring_done + m, 1);  // padding pixel of a partial tile: nothing to trace
          }
        }
        disp_s += give;
        while (disp_s >= spp) { disp_s -= spp; disp_seq++; }
      }
      // set up the segment: invariants + root box test; a root miss is shaded (sky) on the spot and the path ends
      bool go = false;
      if (state == 1) {
        const float4 ro = ray_o[my], rd = ray_d[my];
        Ray r;
        r.o = v3(ro.x, ro.y, ro.z);
        r.d = v3(rd.x, rd.y, rd.z);
        const RayInv q = ray_invariants(r);
        if (box_hit(P.root_box[0], P.root_box[1], P.root_box[2], P.root_box[3], P.root_box[4], P.root_box[5], r, q)) {
          ray_o[my] = make_float4(ro.x, ro.y, ro.z, q.a);
          ray_i[my] = make_float4(q.ix, q.iy, q.iz, 0.0f);
          best_t[my] = kLwNoHit;
          go = true;
        } else {
          const float4 pl = p_light[my];  // miss (ray.fut:141-148)
          V3 light = v3(pl.x, pl.y, pl.z), colour;
          int depth = __float_as_int(pl.w);
          shade_segment(sc, P, r, q.a, -1, 0.0f, light, depth, colour);
          finish_path(my, colour);
          state = 2;
        }
      }
      const unsigned gom = __ballot_sync(kFullMask, go);
      if (go) { ready[nready + __popc(gom & lt_mask)] = (unsigned char)my; state = 0; my = -1; }
      nready += __popc(gom);
      __syncwarp();
      // another pass only helps if some slot has no path and there is still work to hand out
      const bool more = !exhausted || undispensed() > 0;
      if (!more || (!__any_sync(kFullMask, state == 2) && nfree == 0)) break;
    }
    // slots still without a path go (back) to the free list
    const unsigned fm = __ballot_sync(kFullMask, state == 2);
    if (state == 2) freel[nfree + __popc(fm & lt_mask)] = (unsigned char)my;
    nfree += __popc(fm);
    __syncwarp();
  };

  shade_phase();  // first fill
  for (;;) {
    // ---------------------------------------------------------------- lanes between traversals
    const unsigned finm = __ballot_sync(kFullMask, cur == kLwFin);
    if (finm) {
      if (cur == kLwFin) { done[ndone + __popc(finm & lt_mask)] = (unsigned char)(tag >> kSlotShift); cur = kLwIdle; }
      ndone += __popc(finm);
    }
    const unsigned idle = __ballot_sync(kFullMask, cur == kLwIdle);
    if (idle && nready > 0) {
      __syncwarp();
      const int rk = __popc(idle & lt_mask), n = min(__popc(idle), nready);
      if (cur == kLwIdle && rk < n) {
        const int s = ready[nready - 1 - rk];
        const float4 ro = ray_o[s], ri = ray_i[s];
        tag = (uint32_t)s << kSlotShift;
        ox = ro.x; oy = ro.y; oz = ro.z;
        ix = ri.x; iy = ri.y; iz = ri.z;
        cur = 0;
        sp = sbase;
      }
      nready -= n;
    }
    const unsigned act = __ballot_sync(kFullMask, cur >= 0);
    const int n_idle = 32 - __popc(act);
    if (act == 0u || ndone >= 32 || (nready == 0 && ndone > 0 && n_idle >= idle_min)) {
      if (act == 0u && ndone == 0 && nready == 0 && exhausted && undispensed() <= 0 && nfree == R) {
        drain_leaves();  // (nothing can be queued here; kept for symmetry)
        if (kSpread) finalize_pixels();
        if (P.warp_trace && lane == 0) P.warp_trace[1 + blockIdx.x * (blockDim.x >> 5) + warp] = global_timer_ns();
        break;                                                      // frame done for this warp
      }
      __syncwarp();
      drain_leaves();   // every finished traversal's sphere items are folded before its segment is shaded
      shade_phase();
      continue;
    }

    // ---------------------------------------------------------------- one node step per walking lane
    bool l_leaf = false, r_leaf = false;
    int lptr = 0, rptr = 0;
    if (cur >= 0) {
      float4 q0, q1, q2, q3;
      sc.node(cur, q0, q1, q2, q3);
      Ray r;
      r.o = v3(ox, oy, oz);
      r.d = v3(0.0f, 0.0f, 0.0f);
      RayInv q;
      q.ix = ix; q.iy = iy; q.iz = iz; q.a = 0.0f;
      lptr = __float_as_int(q0.w);
      rptr = __float_as_int(q1.w);
      const bool hl = box_hit(q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, r, q);
      const bool hr = box_hit(q2.x, q2.y, q2.z, q3.x, q3.y, q3.z, r, q);
      l_leaf = lptr < 0;             // a leaf child has no box in the reference (bvh.fut:84): always visited
      r_leaf = rptr < 0;
      const bool tl = hl && !l_leaf, tr = hr && !r_leaf;
      if (tl && tr) { *sp = (uint32_t)rptr; sp += 32; }   // left first, right deferred on the private stack
      int nxt = tl ? lptr : rptr;
      if (!(tl || tr)) {
        if (sp != sbase) { sp -= 32; nxt = (int)*sp; }
        else nxt = kLwFin;
      }
      cur = nxt;
    }
    const unsigned cl = __ballot_sync(kFullMask, l_leaf), cr = __ballot_sync(kFullMask, r_leaf);
    if (cl | cr) {
      const int lb = ltop + __popc(cl & lt_mask) + __popc(cr & lt_mask);
      if (l_leaf) lstk[lb] = tag | (uint32_t)(~lptr);
      if (r_leaf) lstk[lb + (l_leaf ? 1 : 0)] = tag | (uint32_t)(~rptr);
      ltop += __popc(cl) + __popc(cr);
      __syncwarp();
      if (ltop >= 32) leaf_batch(32);
      if (ltop >= 32) leaf_batch(32);
    }
  }
  signal_frame_done(P);
}

}  // namespace

cudaError_t launch_lanewalk(const RenderParams &p, const LaunchConfig &lc, cudaStream_t stream, int64_t *launches) {
  const long long items = p.local_tiles * kTilePixels;
  const bool all_nodes = p.smem_nodes == p.n_inner, sph = p.smem_spheres == p.n_leaves && p.smem_spheres > 0;
  const int wthreads = 32 * lc.wq_warps;
  const int scap = lw_stack_capacity(p.max_depth);
  const size_t wsmem = ((staging_bytes(p) + 127) & ~(size_t)127) + (size_t)lc.wq_warps * lw_warp_bytes(lc.lw_slots, scap);
  long long ctas = lc.sm_count;
  const bool spread = p.sample_buf != nullptr;
  // no more CTAs than there are rays to start at once: a slot takes one SAMPLE when samples are spread, one pixel otherwise
  const long long rays = items * (spread ? (long long)p.spp : 1ll);
  const long long per_cta = (long long)lc.lw_slots * lc.wq_warps;
  const long long useful = (rays + per_cta - 1) / per_cta;
  if (ctas > useful) ctas = useful;
  const int idle_min = lc.lw_idle_min < 1 ? 1 : (lc.lw_idle_min > 32 ? 32 : lc.lw_idle_min);
  const int max_pass = lc.lw_passes < 1 ? 1 : lc.lw_passes;
  const auto with_slots = [&](auto slots) {  // the slot counts that are built: 32, 48, 64
    return with_flags([&](auto sp, auto a, auto s) {
      return launch_opted_in<render_lanewalk_kernel<decltype(slots)::value, sp, a, s>>(
          lc.max_dynamic_smem, (unsigned)ctas, wthreads, wsmem, stream, p, scap, idle_min, max_pass);
    }, spread, all_nodes, sph);
  };
  cudaError_t e;
  if (lc.lw_slots == 64) e = with_slots(std::integral_constant<int, 64>{});
  else if (lc.lw_slots == 48) e = with_slots(std::integral_constant<int, 48>{});
  else if (lc.lw_slots == 32) e = with_slots(std::integral_constant<int, 32>{});
  else return cudaErrorInvalidValue;
  if (e == cudaSuccess) (*launches)++;
  return e;
}

#else   // product build: K5 is not compiled in

cudaError_t launch_lanewalk(const RenderParams &, const LaunchConfig &, cudaStream_t, int64_t *) { return cudaErrorNotSupported; }
#endif

}  // namespace rayb200
