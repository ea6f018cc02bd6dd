// Device code shared by the render kernels (render_kernels.cu: K0 mega / K3 warp-queue; render_lanewalk.cu: K5
// lane-walk; render_alt_kernels.cu: the measured-slower alternatives K1 / K2 / K4).  Every translation unit that includes
// this header is compiled with -fmad=false; see device_math.cuh for the bit-exactness rules.
//
// Traversal.  The reference walks the Karras tree stacklessly (parent pointers, bvh.fut:61-84) and
// tests every box against the ORIGINAL ray interval (0, 1e9) (ray.fut:77), so the set of leaves it
// applies `closest_hit` to is exactly { leaf : every ancestor's box passes aabb_hit } - independent
// of traversal order - and the fold result is the leaf with the smallest accepted t, lowest leaf index
// on ties (strict `<` at ray.fut:40 with a shrinking t_max, leaves folded in ascending order).  We
// visit the same set with a left-first stack DFS over the BVH2C layout (scene_host.h): one node step
// tests both children's boxes, ~half the dependent steps of the reference loop and no re-visits.
// See find_closest for how leaf tests are decoupled from the walk and how ties are broken.
#pragma once
#include "render_params.h"
#include "device_math.cuh"

#include <cstdio>
#include <type_traits>

namespace rayb200 {

namespace {

constexpr int kDone = (int)0x80000000;  // traversal sentinel: neither an inner index (>= 0) nor a leaf (~i, i < 2^30)
constexpr unsigned kFullMask = 0xffffffffu;

struct WorkCounters {
  unsigned long long segments = 0, node_steps = 0, box_tests = 0, leaf_tests = 0;
};

// ------------------------------------------------------------------ scene access policies
// A 64-byte node record from global memory as four 128-bit read-only loads (SASS: LDG.E.128.CONSTANT).  128 bits is the
// widest load sm_90 has; the record is 64-byte aligned, so the four loads touch one L1TEX line.
__device__ __forceinline__ void ldg_node(const float4 *p, float4 &q0, float4 &q1, float4 &q2, float4 &q3) {
  q0 = __ldg(p); q1 = __ldg(p + 1); q2 = __ldg(p + 2); q3 = __ldg(p + 3);
}
struct GlobalScene {  // everything through the read-only path (L1/L2)
  const float4 *nodes, *geom;
  __device__ __forceinline__ void node(int cur, float4 &q0, float4 &q1, float4 &q2, float4 &q3) const {
    ldg_node(nodes + 4 * (size_t)cur, q0, q1, q2, q3);
  }
  __device__ __forceinline__ float4 sphere(int i) const { return __ldg(geom + i); }
};

template <bool kAllNodes, bool kSpheres>
struct StagedScene {  // top of the tree (BFS prefix) + optionally all spheres in shared memory
  const float4 *nodes, *geom;
  const float4 *s_nodes, *s_geom;
  int smem_nodes;
  __device__ __forceinline__ void node(int cur, float4 &q0, float4 &q1, float4 &q2, float4 &q3) const {
    if (kAllNodes || cur < smem_nodes) {  // component-major in shared memory: 16-B stride -> all 8 bank groups in play
      const float4 *p = s_nodes + cur;
      q0 = p[0]; q1 = p[smem_nodes]; q2 = p[2 * smem_nodes]; q3 = p[3 * smem_nodes];
    } else {
      ldg_node(nodes + 4 * (size_t)cur, q0, q1, q2, q3);
    }
  }
  __device__ __forceinline__ float4 sphere(int i) const { return kSpheres ? s_geom[i] : __ldg(geom + i); }
};

// ------------------------------------------------------------------ objs_hit, first half (ray.fut:76-82)
// bvh_fold contains closest_hit (-1, 1e9): returns the winning leaf (or -1) and its t.
//
// Because the reference never prunes by the running closest t, node traversal and sphere tests are
// independent: the walk only *collects* the leaves it reaches (a leaf child is recorded by its
// parent's node step, no extra iteration) and the sphere tests run afterwards in a tight loop.  This
// keeps a warp's lanes in the same loop body instead of ping-ponging between "descend" and "test
// leaf".  Collected leaves are not in ascending order any more, so the reference's tie-break (strict
// `<` while folding leaves in ascending index order = lowest index wins an exact t tie) is applied
// explicitly.  sphere_t is evaluated against the ORIGINAL t_max = 1e9: the value sphere_hit returns
// does not depend on the shrinking t_max, only whether it is accepted does (root2 >= root1, so when
// root1 is rejected for being >= t_max, root2 is too).
constexpr int kLeafBuf = 16;

template <bool kCount, class Scene>
__device__ __forceinline__ void test_leaves(const Scene &sc, const int *leaves, int &nl, const Ray &r, const RayInv &q,
                                            int &best_j, float &best_t, WorkCounters &wc) {
  for (int k = 0; k < nl; k++) {
    const int li = leaves[k];
    const float4 g = sc.sphere(li);
    if (kCount) wc.leaf_tests++;
    const float t = sphere_t(g.x, g.y, g.z, g.w, r, q.a, 0.1f, 1000000000.0f);  // closest_hit, ray.fut:78-81
    if (t >= 0.0f && (t < best_t || (t == best_t && li < best_j))) { best_t = t; best_j = li; }
  }
  nl = 0;
}

template <bool kCount, class Scene>
__device__ __forceinline__ void find_closest(const Scene &sc, const float *root_box, const Ray &r, const RayInv &q,
                                             int &best_j, float &best_t, WorkCounters &wc) {
  best_j = -1;
  best_t = 1000000000.0f;
  if (kCount) { wc.segments++; wc.box_tests++; }
  if (!box_hit(root_box[0], root_box[1], root_box[2], root_box[3], root_box[4], root_box[5], r, q)) return;
  int stack[kStackSize + 1];
  int leaves[kLeafBuf];
  int sp = 1, nl = 0;
  stack[0] = kDone;  // popping the sentinel ends the walk
  int cur = 0;
  while (cur != kDone) {
    if (nl > kLeafBuf - 2) test_leaves<kCount>(sc, leaves, nl, r, q, best_j, best_t, wc);
    float4 q0, q1, q2, q3;
    sc.node(cur, q0, q1, q2, q3);
    const int lptr = __float_as_int(q0.w), rptr = __float_as_int(q1.w);
    const bool hl = box_hit(q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, r, q);
    const bool hr = box_hit(q2.x, q2.y, q2.z, q3.x, q3.y, q3.z, r, q);
    const bool l_leaf = lptr < 0, r_leaf = rptr < 0;
    if (kCount) { wc.node_steps++; wc.box_tests += !l_leaf + !r_leaf; }
    // a leaf child has no box in the reference (bvh.fut:84): it is always visited -> record it
    if (l_leaf) leaves[nl] = ~lptr;
    nl += l_leaf;
    if (r_leaf) leaves[nl] = ~rptr;
    nl += r_leaf;
    // inner children whose box is hit are walked: left first, right deferred on the stack
    const bool tl = hl && !l_leaf, tr = hr && !r_leaf;
    if (tl && tr) stack[sp] = rptr;
    sp += (tl && tr);
    int nxt = tl ? lptr : rptr;
    if (!(tl || tr)) nxt = stack[--sp];
    cur = nxt;
  }
  test_leaves<kCount>(sc, leaves, nl, r, q, best_j, best_t, wc);
}

// ------------------------------------------------------------------ one ray_colour iteration (ray.fut:130-148)
// The part of a ray_colour iteration after the closest-hit search: given the fold result (j, tb),
// re-intersect, scatter or shade the sky.  `a` = dot r.d r.d.  Returns true if the path continues
// (r/light/depth updated), false if it ended with `colour` set.  `max_depth`: ray_colour's depth limit (ray.fut:154
// passes 50; a path query passes its own).
template <class Scene>
__device__ __forceinline__ bool shade_segment(const Scene &sc, const RenderParams &P, Ray &r, const float a, const int j,
                                              const float tb, V3 &light, int &depth, V3 &colour,
                                              const int max_depth = kMaxDepth) {
  if (j >= 0) {
    // objs_hit, second half (ray.fut:83-85): re-intersect the winner with t_min = 0, t_max = t_best + 1
    const float4 g = sc.sphere(j);
    const float t = sphere_t(g.x, g.y, g.z, g.w, r, a, 0.0f, tb + 1.0f);
    if (t >= 0.0f) {
      const V3 c = v3(g.x, g.y, g.z);
      const V3 p = vadd(r.o, vscale(t, r.d));                       // point_at_param, ray.fut:14-15
      const V3 n = vscale(1.0f / g.w, vsub(p, c));                  // ray.fut:42-43
      // scatter (ray.fut:119-124): reflect (normalise r.dir) hit.normal; norm r.dir = sqrt(dot d d) = sqrt(a)
      const V3 unit = vscale(1.0f / sqrtf(a), r.d);
      const V3 refl = vsub(unit, vscale(2.0f * vdot(unit, n), n));  // ray.fut:116-117
      if (vdot(refl, n) > 0.0f) {
        const float4 col = __ldg(P.colour + j);
        r.o = p;
        r.d = refl;
        light = vmul(light, v3(col.x, col.y, col.z));               // ray.fut:135
        depth = depth + 1;
        if (depth < max_depth) return true;
        colour = v3(0.0f, 0.0f, 0.0f);                              // loop exit with colour = light*0 (ray.fut:136)
        return false;
      }
      colour = v3(0.0f, 0.0f, 0.0f);                                // ray.fut:137-140
      return false;
    }
  }
  // miss: sky gradient (ray.fut:141-148)
  const V3 unit = vscale(1.0f / sqrtf(a), r.d);
  const float t = 0.5f * (unit.y + 1.0f);
  const float w1 = 1.0f - t;
  const V3 sky = v3(w1 * 1.0f + t * 0.5f, w1 * 1.0f + t * 0.7f, w1 * 1.0f + t * 1.0f);
  colour = vmul(light, sky);
  return false;
}

// One whole ray_colour iteration for a lane-owned path.  `depth` counts objs_hit calls so far (ray.fut:129).
template <bool kCount, class Scene>
__device__ __forceinline__ bool advance_path(const Scene &sc, const RenderParams &P, Ray &r, V3 &light, int &depth,
                                             V3 &colour, WorkCounters &wc) {
  const RayInv q = ray_invariants(r);
  int j;
  float tb;
  find_closest<kCount>(sc, P.root_box, r, q, j, tb, wc);
  return shade_segment(sc, P, r, q.a, j, tb, light, depth, colour);
}

// get_ray (ray.fut:109-114) of camera c (origin, llc, horizontal, vertical) at (u, v)
__device__ __forceinline__ Ray camera_ray(const float *c, const float u, const float v) {
  Ray r;
  r.o = v3(c[0], c[1], c[2]);
  // llc + s*horizontal + t*vertical - origin (ray.fut:111-113), per component, left to right
  r.d = v3(((c[3] + u * c[6]) + v * c[9]) - c[0], ((c[4] + u * c[7]) + v * c[10]) - c[1],
           ((c[5] + u * c[8]) + v * c[11]) - c[2]);
  return r;
}

// get_ray for sample s of pixel (row j, column i): ray.fut:150-154 with pixel j i -> trace_ray (height-j) i
// (ray.fut:167-168) and the spp extension of ray_b200.h (offset (0,0) at s = 0).  kAccum (a chunk of a progressive frame):
// s is relative to the chunk, P.offsets starts at its first sample and is read even when P.spp == 1; at s = 0 of the
// frame the offset is (0, 0) and f32(i) + 0 is exact, so that is the one-sample ray too.  kViews (a views launch): the
// camera is view_cam, the pixel's view's 12 floats of RayQuery::cams, instead of P.cam.
template <bool kAccum = false, bool kViews = false>
__device__ __forceinline__ Ray primary_ray(const RenderParams &P, int i, int j, int s, const float *view_cam = nullptr) {
  float u, v;
  if (!kAccum && P.spp == 1) {
    u = (float)i / (float)P.W;
    v = (float)(P.H - j) / (float)P.H;
  } else {
    u = ((float)i + P.offsets[2 * s]) / (float)P.W;
    v = ((float)(P.H - j) + P.offsets[2 * s + 1]) / (float)P.H;
  }
  if constexpr (kViews) {  // three 16-byte read-only loads (the table is 16-byte aligned, 48 bytes per view)
    const float4 *q = reinterpret_cast<const float4 *>(view_cam);
    const float4 a = __ldg(q), b = __ldg(q + 1), d = __ldg(q + 2);
    const float c[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, d.x, d.y, d.z, d.w};
    return camera_ray(c, u, v);
  }
  return camera_ray(P.cam, u, v);
}

// item k -> pixel.  Local tile lt = k >> 5 is global tile lt*world + rank; lane position k & 31 inside the 8x4 tile.
// (fill_params caps a frame at 2^25 tiles, so the global tile index fits 32 bits: one 32-bit division instead of the
// 64-bit one, which is a ~100-instruction subroutine executed at ~3 of 32 lanes on the refill / finish paths.)
__device__ __forceinline__ bool item_pixel(const RenderParams &P, int k, int &i, int &j) {
  const unsigned t = (unsigned)(k >> 5) * (unsigned)P.world + (unsigned)P.rank;
  const int sub = k & 31;
  const unsigned ty = t / (unsigned)P.tiles_x, tx = t - ty * (unsigned)P.tiles_x;
  i = (int)tx * kTileW + (sub & (kTileW - 1));
  j = (int)ty * kTileH + (sub >> 3);
  return (long long)t < P.n_tiles && i < P.W && j < P.H;
}

// kViews: item k -> view v and pixel.  The views' tiles follow each other, view_tiles = tiles_x * tiles_y per view in the
// row-major tile order of one frame (a views launch has no shards).  Tile t is in tile row r = t / tiles_x over all
// views, which is row r - v * tiles_y of view v = r / tiles_y: two 32-bit divisions (n_tiles <= 2^25).
__device__ __forceinline__ bool item_view_pixel(const RenderParams &P, int k, int &v, int &i, int &j) {
  const unsigned t = (unsigned)(k >> 5);
  const int sub = k & 31;
  const unsigned r = t / (unsigned)P.tiles_x, tx = t - r * (unsigned)P.tiles_x;
  const unsigned vv = r / (unsigned)P.tiles_y, ty = r - vv * (unsigned)P.tiles_y;
  v = (int)vv;
  i = (int)tx * kTileW + (sub & (kTileW - 1));
  j = (int)ty * kTileH + (sub >> 3);
  return (long long)t < P.n_tiles && i < P.W && j < P.H;
}

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// claim index (value of the global work cursor) -> item index: chunks of 64 tiles in stride-permuted order
__device__ __forceinline__ int claim_to_item(const RenderParams &P, int c) {
  if (P.tile_order) {  // heavy-first order from the probe pass
    const int lt = c >> 5;
    return lt < P.local_tiles ? (__ldg(P.tile_order + lt) << 5) | (c & 31) : (int)(P.local_tiles << 5);
  }
  const int chunk = c >> 11;
  const int perm = (int)(((long long)chunk * P.chunk_stride) % P.n_chunks);
  return (perm << 11) | (c & 2047);
}

// kAccum: the sum of a progressive frame's samples [0, s_end), always scaled by P.inv_spp = 1/s_end (1 * x = x when
// s_end = 1; a NaN stays some NaN), and the pixel frame is optional (row-major only).  kViews: pixel (i, j) of view
// `view`, whose frames follow each other (row-major; 64-bit offsets: V x H x W reaches 2^30, the float frames 12 GiB)
template <bool kAccum = false, bool kViews = false>
__device__ __forceinline__ void write_pixel(const RenderParams &P, int k, int i, int j, V3 sum, int view = 0) {
  const V3 col = (!kAccum && P.spp == 1) ? sum : vscale(P.inv_spp, sum);
  const int pix = pack_pixel(col);
  if constexpr (kViews) {
    const size_t px = (size_t)view * (size_t)P.H * (size_t)P.W + (size_t)j * P.W + i;
    P.out_pix[px] = pix;
    if (P.out_rgb) {
      float *q = P.out_rgb + 3 * px;
      q[0] = col.x; q[1] = col.y; q[2] = col.z;
    }
    return;
  }
  if constexpr (kAccum) {
    if (P.out_pix) P.out_pix[(size_t)j * P.W + i] = pix;
  } else if (P.tile_major) {
    P.out_pix[k] = pix;
  } else {
    P.out_pix[(size_t)j * P.W + i] = pix;
  }
  if (P.out_rgb) {
    float *q = P.out_rgb + 3 * ((size_t)j * P.W + i);
    q[0] = col.x; q[1] = col.y; q[2] = col.z;
  }
}

// Peer-frame protocol: called by every warp as it leaves a persistent kernel (all lanes).  The warp's pixel stores may
// have gone to another GPU's memory over NVLink; the last warp of the launch publishes "this rank's part of the frame
// has landed" by bumping the consumer's flag — fence first, so the flag can never overtake the pixels.
__device__ __forceinline__ void signal_frame_done(const RenderParams &P) {
  if (P.frame_flag == nullptr) return;
  __syncwarp();
  if ((threadIdx.x & 31) == 0) {
    __threadfence_system();
    const int total_warps = (int)(gridDim.x * (blockDim.x >> 5));
    if (atomicAdd(P.work_cursor + 1, 1) == total_warps - 1) {
      __threadfence_system();
      atomicAdd_system(P.frame_flag, 1u);
    }
  }
}

__device__ __forceinline__ void flush_counters(const RenderParams &P, WorkCounters &wc) {
  for (int o = 16; o > 0; o >>= 1) {
    wc.segments += __shfl_down_sync(kFullMask, wc.segments, o);
    wc.node_steps += __shfl_down_sync(kFullMask, wc.node_steps, o);
    wc.box_tests += __shfl_down_sync(kFullMask, wc.box_tests, o);
    wc.leaf_tests += __shfl_down_sync(kFullMask, wc.leaf_tests, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(P.counters + 0, wc.segments);
    atomicAdd(P.counters + 1, wc.node_steps);
    atomicAdd(P.counters + 2, wc.box_tests);
    atomicAdd(P.counters + 3, wc.leaf_tests);
  }
}

// ====================================================================================== closest-hit fold (item kernels)
// K3 / K5 test (ray, sphere) items in dense batches, any lane for any ray, so a slot's closest hit is folded in shared
// memory: "smallest t, lowest Morton-sorted leaf index on ties" (ray.fut:40's strict `<` over leaves folded in
// ascending order).  A 64-bit atomicMin on (bits(t) << 32 | leaf) does that in one operation but is a CAS loop in
// shared memory (ATOMS.CAST.SPIN); this is the same fold with
// native 32-bit ATOMS.MIN: t first, then the leaf among the lanes that hold the final t.  Positive floats order like
// their bit patterns; kItemNoHit (all ones) is above every t < 1e9.  Warp-collective: call with all 32 lanes.
constexpr int kSlotShift = 26;                 // item = slot << 26 | index  (index < 2^26; R <= 64 slots)
constexpr uint32_t kIndexMask = (1u << kSlotShift) - 1u;
constexpr uint32_t kItemNoHit = 0xffffffffu;

__device__ __forceinline__ void fold_hit(uint32_t *best_t, uint32_t *best_l, const int slot, const bool hit, const uint32_t tb,
                                         const uint32_t li) {
  uint32_t old = 0u;
  if (hit) old = atomicMin(best_t + slot, tb);
  __syncwarp();
  // the lanes that hold the slot's minimum after this batch: exactly one of them lowered it (old > tb) unless the
  // minimum is not new, the others tie with a value that was already there (set in this batch or an earlier one)
  const bool mine = hit && *reinterpret_cast<volatile uint32_t *>(best_t + slot) == tb;
  const bool tie = mine && old == tb;
  if (mine && old > tb) best_l[slot] = li;
  if (__any_sync(kFullMask, tie)) {
    __syncwarp();
    if (tie) atomicMin(best_l + slot, li);
  }
  __syncwarp();
}

// ====================================================================================== TMA staging helpers
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_addr(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// 1-D bulk async copy global -> shared through the TMA unit (SASS: UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_addr(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}

// Stages the BFS prefix of the node array (and optionally all sphere records) into shared memory.
// One elected thread arms the mbarrier with the byte count and issues the bulk copies; everyone waits on it.
__device__ __forceinline__ void stage_scene(const RenderParams &P, unsigned char *smem_raw, const float4 *&s_nodes,
                                            const float4 *&s_geom) {
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
  float4 *nodes_dst = reinterpret_cast<float4 *>(smem_raw + 128);
  float4 *geom_dst = nodes_dst + 4 * (size_t)P.smem_nodes;
  const uint32_t node_bytes = (uint32_t)P.smem_nodes * 64u, geom_bytes = (uint32_t)P.smem_spheres * 16u;
  if (threadIdx.x == 0) mbar_init(bar, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, node_bytes + geom_bytes);
    constexpr uint32_t kChunk = 32768;
    // component-major: the first smem_nodes entries of each of the four component arrays
    const uint32_t comp_bytes = (uint32_t)P.smem_nodes * 16u;
    for (int c = 0; c < 4; c++)
      for (uint32_t off = 0; off < comp_bytes; off += kChunk)
        tma_bulk_g2s(reinterpret_cast<unsigned char *>(nodes_dst + (size_t)c * P.smem_nodes) + off,
                     reinterpret_cast<const unsigned char *>(P.nodes_soa + (size_t)c * P.n_inner) + off,
                     min(kChunk, comp_bytes - off), bar);
    for (uint32_t off = 0; off < geom_bytes; off += kChunk)
      tma_bulk_g2s(reinterpret_cast<unsigned char *>(geom_dst) + off, reinterpret_cast<const unsigned char *>(P.geom) + off,
                   min(kChunk, geom_bytes - off), bar);
  }
  mbar_wait(bar, 0);
  s_nodes = nodes_dst;
  s_geom = geom_dst;
}

// Opt a kernel in to `max_dynamic_smem` bytes of dynamic shared memory, once per (instantiation, device).
template <auto Kern>
cudaError_t opt_in_dynamic_smem(int max_dynamic_smem) {
  static bool done_for[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (done_for[dev & 63]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_dynamic_smem);
  if (e == cudaSuccess) done_for[dev & 63] = true;
  return e;
}

// Variant dispatch of the host launchers: with_flags(f, b0, b1, ...) calls f(std::bool_constant<b0>{}, ...), so run-time
// flags pick compile-time template arguments.  f is instantiated for every combination of the flags passed, so a
// launcher passes only axes whose combinations all exist (K3's ray-mode axes are dispatched apart from its pixel axes).
template <class F>
cudaError_t with_flags(F &&f) { return f(); }
template <class F, class... B>
cudaError_t with_flags(F &&f, bool b, B... rest) {
  if (b) return with_flags([&](auto... c) { return f(std::true_type{}, c...); }, rest...);
  return with_flags([&](auto... c) { return f(std::false_type{}, c...); }, rest...);
}
// ... and with_query(f, q) calls f(std::integral_constant<Query, q>{}) for the ray-query kinds (Query::kPixels is not one)
template <class F>
cudaError_t with_query(F &&f, Query q) {
  switch (q) {
    case Query::kClosest: return f(std::integral_constant<Query, Query::kClosest>{});
    case Query::kAnyHit: return f(std::integral_constant<Query, Query::kAnyHit>{});
    case Query::kMultiHit: return f(std::integral_constant<Query, Query::kMultiHit>{});
    default: return cudaErrorInvalidValue;
  }
}

// Opts Kern in to the device's dynamic shared memory on first use, then launches it.
template <auto Kern, class... Args>
cudaError_t launch_opted_in(int max_dynamic_smem, unsigned grid, int block, size_t smem, cudaStream_t stream, const Args &...args) {
  const cudaError_t e = opt_in_dynamic_smem<Kern>(max_dynamic_smem);
  if (e == cudaSuccess) Kern<<<grid, block, smem, stream>>>(args...);
  return e;
}

}  // namespace

}  // namespace rayb200
