// Device-side prepare_scene (SURVEY.md §8f row N1): the reference's bvh_mk (futhark/bvh.fut:30-59) and
// mk_radix_tree (futhark/radixtree.fut:11-72) as sm_90a kernels, producing bit-identical arrays to the
// host builder in scene_host.cpp (tests/test_gpu_parity.py compares the two) and the packed BVH2C layout
// the render kernels walk.  Compiled with -fmad=false like every other f32 in this library.
//
//   centres + 6 min/max reductions   bvh.fut:31-37     one kernel (shuffle reduce + ordered-int atomics)
//   Morton keys                      bvh.fut:38-41,8-22 one kernel
//   stable sort by key               bvh.fut:43        cub::DeviceRadixSort::SortPairs (LSD radix sort = stable, like
//                                                       the reference's radix_sort_by_key, radix_sort.fut:50-68)
//   Karras radix tree                radixtree.fut     one kernel, one thread per inner node; parents by scatter
//   fixed-count Jacobi refit         bvh.fut:44-58     trunc(log2 n)+2 launches, ping-pong boxes (NOT run to convergence:
//                                                       the reference renders with the stale boxes this leaves)
//   layout                           (ours)            node depth by parent walk, stable sort by depth (= order by
//                                                       (depth, Karras index), the same order pack_bvh uses), pack
//
// Scene batches (DESIGN.md §5b): B scenes of n_0 .. n_{B-1} spheres, back to back in one sphere array, are built in the
// same launches.  Scene b's leaves start at off[b] = n_0 + .. + n_{b-1} and its inner nodes at off[b] - b, so one table
// off[B + 1] places both, and every kernel finds its element's scene in it (scene_of, an upper-bound search).  One box
// per scene for the Morton keys, one stable sort on (scene << 32 | key), which is each scene's own stable sort, the radix
// tree of each scene's key segment with global child, leaf and parent indices, each scene's own number of refit sweeps
// (a scene whose sweeps are done copies its boxes through the remaining ones), and one stable sort on (scene, depth) for
// the layout, so scene b's nodes are one block in its own (depth, Karras index) order and its root is node off[b] - b.
// B = 1 is the single-scene build, with its 32-bit key sorts.
#include "bvh_build.h"

#include <cub/cub.cuh>

#include <cmath>

namespace rayb200 {

namespace {

constexpr int kThreads = 256;
inline unsigned blocks_for(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// order-preserving float <-> int maps for atomicMin/atomicMax on floats (inputs are never NaN here)
__device__ __forceinline__ int float_to_ordered(float f) {
  const int b = __float_as_int(f);
  return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

struct SphereBox {
  float lo[3], hi[3];
};
// sphere_aabb (ray.fut:28-30)
__device__ __forceinline__ SphereBox sphere_box(const float *sp) {
  SphereBox b;
  const float r = sp[6];
  b.lo[0] = sp[0] - r; b.lo[1] = sp[1] - r; b.lo[2] = sp[2] - r;
  b.hi[0] = sp[0] + r; b.hi[1] = sp[1] + r; b.hi[2] = sp[2] + r;
  return b;
}

// Where the scenes of a build start: `count` scenes whose leaves start at off[b] (device [count + 1]; NULL for one scene)
// and whose inner nodes start at off[b] - b.  n_uni > 0: every scene has n_uni leaves (off[b] = b n_uni), which the
// kernels compute instead of searching the table.
struct Scenes {
  const int32_t *off;
  int count, n_uni;
};
// The scene of leaf k (inner = 0) or inner node k (inner = 1): the last b whose first element is <= k.  One scene: 0.
__device__ __forceinline__ int scene_of(const Scenes S, int k, int inner) {
  if (S.n_uni > 0) return k / (S.n_uni - inner);
  int lo = 0, hi = S.count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(S.off + mid) - inner * mid <= k) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}
// The first leaf of scene sc (off[sc])
__device__ __forceinline__ int leaf_start(const Scenes S, int sc) { return S.n_uni > 0 ? sc * S.n_uni : __ldg(S.off + sc); }

// Identity elements of the min / max reductions, as ordered ints (any real float beats them), and zeroed per-scene
// results: minmax [scenes][6], result [scenes][2]
__global__ void init_build_kernel(int *__restrict__ minmax, int *__restrict__ result, int scenes) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < scenes; s += gridDim.x * blockDim.x) {
    for (int a = 0; a < 3; a++) { minmax[6 * (size_t)s + a] = 0x7fffffff; minmax[6 * (size_t)s + 3 + a] = (int)0x80000000; }
    result[2 * (size_t)s] = 0;
    result[2 * (size_t)s + 1] = 0;
  }
}

// bvh.fut:31-37: centre of every sphere box (prim.fut:47-50) and the six min/max reductions over them, per scene.  Warp
// w takes spheres [w per_warp, (w + 1) per_warp) of all scenes' `total`, 32 at a time, so the grid follows the total
// whatever the counts.  While a warp's spheres stay in one scene its lanes reduce in registers; a step that straddles
// scenes is reduced per scene segment (a scene's spheres are contiguous), and the first lane of a segment folds it into
// its scene's min / max.  Min and max are exact in any order.
__global__ void centres_minmax_kernel(const float *__restrict__ spheres, const Scenes S, int total,
                                      int per_warp, float *__restrict__ cx, float *__restrict__ cy, float *__restrict__ cz,
                                      int *__restrict__ minmax /* [scenes][6] ordered ints */) {
  const int lane = threadIdx.x & 31;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w * per_warp >= total) return;  // (whole warps)
  const int begin = (int)(w * per_warp), end = min(total, begin + per_warp);
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  int cur = -1;  // warp-uniform: the scene lo / hi are reducing, -1 = none
  auto fold = [&](int sc, bool first) {  // lane `first` of each segment of equal sc: fold its lo / hi into scene sc's
    if (!first) return;
    for (int a = 0; a < 3; a++) {
      atomicMin(minmax + 6 * (size_t)sc + a, float_to_ordered(lo[a]));
      atomicMax(minmax + 6 * (size_t)sc + 3 + a, float_to_ordered(hi[a]));
    }
  };
  auto reset = [&]() { for (int a = 0; a < 3; a++) { lo[a] = INFINITY; hi[a] = -INFINITY; } };
  auto flush = [&]() {  // the whole warp holds scene cur's partial min / max
    for (int a = 0; a < 3; a++)
      for (int o = 16; o > 0; o >>= 1) {
        lo[a] = fminf(lo[a], __shfl_down_sync(0xffffffffu, lo[a], o));
        hi[a] = fmaxf(hi[a], __shfl_down_sync(0xffffffffu, hi[a], o));
      }
    fold(cur, lane == 0);
    reset();
    cur = -1;
  };
  for (int base = begin; base < end; base += 32) {
    const int k = base + lane;
    const bool live = k < end;
    const int sc = live ? scene_of(S, k, 0) : -1;
    float c[3] = {INFINITY, INFINITY, INFINITY};
    if (live) {
      const SphereBox b = sphere_box(spheres + 7 * (size_t)k);
      c[0] = b.lo[0] + 0.5f * (b.hi[0] - b.lo[0]); c[1] = b.lo[1] + 0.5f * (b.hi[1] - b.lo[1]); c[2] = b.lo[2] + 0.5f * (b.hi[2] - b.lo[2]);
      cx[k] = c[0]; cy[k] = c[1]; cz[k] = c[2];
    }
    const int sc0 = __shfl_sync(0xffffffffu, sc, 0);
    const bool one = __all_sync(0xffffffffu, sc == sc0);
    if (!(one && sc0 == cur) && cur >= 0) flush();
    if (one) {
      cur = sc0;
      for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], c[a]); hi[a] = fmaxf(hi[a], c[a]); }
      continue;
    }
    // a step across scenes: lane i ends with the min / max of [i, its segment's end).  Seeded through fminf / fmaxf from
    // the identities, as every other fold here, so a NaN centre (NaN coordinates, or -inf + inf from a huge radius) is
    // skipped, as the reference's f32.minimum / maximum skip it, and never reaches its scene's box.
    for (int a = 0; a < 3; a++) { lo[a] = fminf(INFINITY, c[a]); hi[a] = fmaxf(-INFINITY, live ? c[a] : -INFINITY); }
    for (int o = 1; o < 32; o <<= 1) {
      const int osc = __shfl_down_sync(0xffffffffu, sc, o);
      for (int a = 0; a < 3; a++) {
        const float l = __shfl_down_sync(0xffffffffu, lo[a], o), h = __shfl_down_sync(0xffffffffu, hi[a], o);
        if (lane + o < 32 && osc == sc) { lo[a] = fminf(lo[a], l); hi[a] = fmaxf(hi[a], h); }
      }
    }
    const int prev = __shfl_up_sync(0xffffffffu, sc, 1);
    fold(sc, live && (lane == 0 || prev != sc));
    reset();
  }
  if (cur >= 0) flush();
}

__device__ __forceinline__ uint32_t spread10(uint32_t v) {  // expand_bits, bvh.fut:8-13
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}
__device__ __forceinline__ uint32_t quantise10(float t) {  // bvh.fut:16-18; NaN (0/0 on a flat axis) -> 0 through fmaxf
  return (uint32_t)fminf(fmaxf(t * 1024.0f, 0.0f), 1023.0f);
}

// bvh.fut:38-41 + morton_3D (bvh.fut:15-22) over `total` spheres, with the box of each sphere's scene (scene_of).
// A batch (key64 != NULL) writes the scene above the key: sorting (scene, key) stably sorts every scene on its own.
__global__ void morton_kernel(const float *__restrict__ cx, const float *__restrict__ cy, const float *__restrict__ cz, int total,
                              const Scenes S, const int *__restrict__ minmax_all, uint32_t *__restrict__ key,
                              uint64_t *__restrict__ key64, int32_t *__restrict__ idx) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= total) return;
  const int sc = scene_of(S, k, 0);
  const int *minmax = minmax_all + 6 * (size_t)sc;
  const float lo[3] = {ordered_to_float(minmax[0]), ordered_to_float(minmax[1]), ordered_to_float(minmax[2])};
  const float hi[3] = {ordered_to_float(minmax[3]), ordered_to_float(minmax[4]), ordered_to_float(minmax[5])};
  const uint32_t qx = quantise10((cx[k] - lo[0]) / (hi[0] - lo[0]));
  const uint32_t qy = quantise10((cy[k] - lo[1]) / (hi[1] - lo[1]));
  const uint32_t qz = quantise10((cz[k] - lo[2]) / (hi[2] - lo[2]));
  const uint32_t m = spread10(qx) * 4u + spread10(qy) * 2u + spread10(qz);
  if (key64) key64[k] = (uint64_t)sc << 32 | m;
  else key[k] = m;
  idx[k] = k;
}

// a batch's sorted (scene, key) pairs -> the 32-bit keys the radix tree reads
__global__ void low_keys_kernel(const uint64_t *__restrict__ key64, int total, uint32_t *__restrict__ key) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < total) key[k] = (uint32_t)key64[k];
}

// mk_radix_tree (radixtree.fut:11-72): one thread per inner node of `scenes` trees over `total` keys (scene_of; one
// scene: n = total).  Scene sc's thread i works on its scene's n keys with local indices and writes global ones: inner
// node i -> off[sc] - sc + i, leaf i -> off[sc] + i.  node_scene (NULL for one scene) gets every inner node's scene.
__global__ void karras_kernel(const uint32_t *__restrict__ M_all, const Scenes S, int total,
                              int32_t *__restrict__ left, int32_t *__restrict__ right, int32_t *__restrict__ parent,
                              int32_t *__restrict__ node_scene) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total - S.count) return;
  const int sc = scene_of(S, g, 1);
  const int leaf0 = S.count == 1 ? 0 : leaf_start(S, sc), n = S.count == 1 ? total : leaf_start(S, sc + 1) - leaf0;
  const int inner0 = leaf0 - sc, i = g - inner0;
  if (node_scene) node_scene[g] = sc;
  const uint32_t *M = M_all + leaf0;
  auto delta = [&](int a, int b) -> int {  // radixtree.fut:13-21
    if (b < 0 || b >= n) return -1;
    const uint32_t x = M[a], y = M[b];
    if (x != y) return __clz((int)(x ^ y));
    return 32 + __clz(a ^ b);
  };
  const int up = delta(i, i + 1), down = delta(i, i - 1);
  const int d = (up > down) - (up < down);                       // :27
  const int floor_cp = delta(i, i - d);                          // :30
  int span = 2;                                                  // :31-33
  while (delta(i, i + span * d) > floor_cp) span *= 2;
  int len = 0;                                                   // :36-40
  for (int step = span / 2; step > 0; step /= 2)
    if (delta(i, i + (len + step) * d) > floor_cp) len += step;
  const int j = i + len * d;                                     // :41
  const int node_cp = delta(i, j);                               // :44
  int split = 0;                                                 // :45-50
  for (int q = 1; q <= len; q *= 2) {
    const int step = (len + q * 2 - 1) / (q * 2);
    if (delta(i, i + (split + step) * d) > node_cp) split += step;
  }
  const int gamma = i + split * d + min(d, 0);                   // :51
  const int l = (min(i, j) == gamma) ? ~(leaf0 + gamma) : inner0 + gamma;             // :54-57
  const int r = (max(i, j) == gamma + 1) ? ~(leaf0 + gamma + 1) : inner0 + gamma + 1;  // :59-62
  left[g] = l;
  right[g] = r;
  if (l >= 0) parent[l] = g;                                     // :66-70 (scatter; the root keeps -1)
  if (r >= 0) parent[r] = g;
}

// The min / max of enclosing (prim.fut:38-45) with -0.0 below +0.0, as the host builder and the oracle define it:
// fminf / fmaxf leave the sign of a min or max of -0.0 and +0.0 open.
__device__ __forceinline__ float min_num(float a, float b) { return a == b ? (signbit(a) ? a : b) : fminf(a, b); }
__device__ __forceinline__ float max_num(float a, float b) { return a == b ? (signbit(a) ? b : a) : fmaxf(a, b); }

__device__ __forceinline__ void child_box(const float *__restrict__ boxes, const float *__restrict__ spheres,
                                          const int32_t *__restrict__ perm, int p, float *b) {
  if (p < 0) {  // leaf: sphere_aabb of L[~p]
    const SphereBox s = sphere_box(spheres + 7 * (size_t)perm[~p]);
    b[0] = s.lo[0]; b[1] = s.lo[1]; b[2] = s.lo[2]; b[3] = s.hi[0]; b[4] = s.hi[1]; b[5] = s.hi[2];
  } else {
    const float *q = boxes + 6 * (size_t)p;
    for (int c = 0; c < 6; c++) b[c] = q[c];
  }
}

// one Jacobi sweep of bvh.fut:52-58: new boxes from the OLD boxes of the children.  Sweep `sweep` of a batch whose scenes
// refit for different counts (sweeps != NULL: scene b's count sweeps[b], node k's scene node_scene[k]): a node whose
// scene has done its own sweeps keeps its box, copied from src to dst, so the last sweep still lands every box in dst.
__global__ void refit_kernel(const float *__restrict__ src, float *__restrict__ dst, const int32_t *__restrict__ left,
                             const int32_t *__restrict__ right, const float *__restrict__ spheres, const int32_t *__restrict__ perm,
                             int ni, const int32_t *__restrict__ sweeps, const int32_t *__restrict__ node_scene, int sweep) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ni) return;
  if (sweeps && sweep >= __ldg(sweeps + node_scene[k])) {
    for (int c = 0; c < 6; c++) dst[6 * (size_t)k + c] = src[6 * (size_t)k + c];
    return;
  }
  float a[6], b[6];
  child_box(src, spheres, perm, left[k], a);
  child_box(src, spheres, perm, right[k], b);
  float *o = dst + 6 * (size_t)k;
  for (int c = 0; c < 3; c++) { o[c] = min_num(a[c], b[c]); o[3 + c] = max_num(a[3 + c], b[3 + c]); }  // enclosing, prim.fut:38-45
}

// diagnostics + layout keys: depth of every inner node (root = 0) and how many boxes are not the union of their children,
// per scene (node_scene, NULL for one scene).  A batch (key64 != NULL) writes (scene, depth) as the layout key.
__global__ void depth_stale_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ left, const int32_t *__restrict__ right,
                                   const int32_t *__restrict__ parent, const float *__restrict__ spheres, const int32_t *__restrict__ perm,
                                   int ni, const int32_t *__restrict__ node_scene, uint32_t *__restrict__ depth, uint64_t *__restrict__ key64,
                                   int32_t *__restrict__ node_id, int *__restrict__ result_all /* [scenes][2]: max depth, stale */) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ni) return;
  const int sc = node_scene ? node_scene[k] : 0;
  int *result = result_all + 2 * (size_t)sc;
  int d = 0;
  for (int p = parent[k]; p >= 0; p = parent[p]) d++;
  if (key64) key64[k] = (uint64_t)sc << 8 | (uint32_t)d;
  else depth[k] = (uint32_t)d;
  node_id[k] = k;
  atomicMax(result, d + 1);  // + the leaf level
  float a[6], b[6];
  child_box(boxes, spheres, perm, left[k], a);
  child_box(boxes, spheres, perm, right[k], b);
  const float *q = boxes + 6 * (size_t)k;
  bool same = true;
  for (int c = 0; c < 3; c++) {
    same = same && __float_as_int(min_num(a[c], b[c])) == __float_as_int(q[c]);
    same = same && __float_as_int(max_num(a[3 + c], b[3 + c])) == __float_as_int(q[3 + c]);
  }
  if (!same) atomicAdd(result + 1, 1);
}

__global__ void invert_kernel(const int32_t *__restrict__ order, int ni, int32_t *__restrict__ newidx) {
  const int pos = blockIdx.x * blockDim.x + threadIdx.x;
  if (pos < ni) newidx[order[pos]] = pos;
}

// BVH2C records (scene_host.h), node-major and component-major copies
__global__ void pack_nodes_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ left, const int32_t *__restrict__ right,
                                  const int32_t *__restrict__ order, const int32_t *__restrict__ newidx, int ni,
                                  float4 *__restrict__ nodes, float4 *__restrict__ soa) {
  const int pos = blockIdx.x * blockDim.x + threadIdx.x;
  if (pos >= ni) return;
  const int k = order[pos];
  const int ch[2] = {left[k], right[k]};
  float4 q[4];
  int ptr[2];
  for (int c = 0; c < 2; c++) {
    if (ch[c] < 0) {  // leaf child: no box in the reference -> always-pass box
      q[2 * c] = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
      q[2 * c + 1] = make_float4(INFINITY, INFINITY, INFINITY, 0.0f);
      ptr[c] = ch[c];
    } else {
      const float *b = boxes + 6 * (size_t)ch[c];
      q[2 * c] = make_float4(b[0], b[1], b[2], 0.0f);
      q[2 * c + 1] = make_float4(b[3], b[4], b[5], 0.0f);
      ptr[c] = newidx[ch[c]];
    }
  }
  q[0].w = __int_as_float(ptr[0]);
  q[1].w = __int_as_float(ptr[1]);
  for (int c = 0; c < 4; c++) {
    nodes[4 * (size_t)pos + c] = q[c];
    soa[(size_t)c * ni + pos] = q[c];
  }
}

__global__ void pack_spheres_kernel(const float *__restrict__ spheres, const int32_t *__restrict__ perm, int n,
                                    float4 *__restrict__ geom, float4 *__restrict__ colour) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float *s = spheres + 7 * (size_t)perm[k];
  geom[k] = make_float4(s[0], s[1], s[2], s[6]);
  colour[k] = make_float4(s[3], s[4], s[5], 0.0f);
}

// pack_spheres_kernel backwards: every record back at its caller-order index (gather_spheres_device)
__global__ void gather_spheres_kernel(const float4 *__restrict__ geom, const float4 *__restrict__ colour,
                                      const int32_t *__restrict__ perm, int64_t n, float *__restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float4 g = geom[k], c = colour[k];
  float *s = out + 7 * (int64_t)perm[k];
  s[0] = g.x; s[1] = g.y; s[2] = g.z;
  s[3] = c.x; s[4] = c.y; s[5] = c.z;
  s[6] = g.w;
}

// per scene: its root box (its Karras root, inner node off[sc] - sc), depth and stale count
__global__ void finish_kernel(const float *__restrict__ boxes, const int *__restrict__ result, const Scenes S,
                              BvhBuildResult *__restrict__ out) {
  const int scenes = S.count;
  for (int sc = blockIdx.x * blockDim.x + threadIdx.x; sc < scenes; sc += gridDim.x * blockDim.x) {
    const float *b = boxes + 6 * (size_t)(scenes == 1 ? 0 : leaf_start(S, sc) - sc);
    for (int c = 0; c < 6; c++) out[sc].root_box[c] = b[c];
    out[sc].max_depth = result[2 * (size_t)sc];
    out[sc].stale_nodes = result[2 * (size_t)sc + 1];
  }
}

// Scene s of a batch as a scene of its own: its blocks of every array, indices made local to it
__device__ __forceinline__ int32_t local_ptr(int32_t p, int32_t inner0, int32_t leaf0) { return p >= 0 ? p - inner0 : ~(~p - leaf0); }

__global__ void extract_scene_kernel(const DeviceBvh src, int32_t s, int32_t off_s, int n, const DeviceBvh dst) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int ni = n - 1, inner0 = off_s - s, leaf0 = off_s;
  if (k < ni) {
    float4 q[4];
    for (int c = 0; c < 4; c++) q[c] = src.nodes[4 * ((size_t)inner0 + k) + c];
    q[0].w = __int_as_float(local_ptr(__float_as_int(q[0].w), inner0, leaf0));
    q[1].w = __int_as_float(local_ptr(__float_as_int(q[1].w), inner0, leaf0));
    for (int c = 0; c < 4; c++) {
      dst.nodes[4 * (size_t)k + c] = q[c];
      dst.nodes_soa[(size_t)c * ni + k] = q[c];
    }
    dst.left[k] = local_ptr(src.left[inner0 + k], inner0, leaf0);
    dst.right[k] = local_ptr(src.right[inner0 + k], inner0, leaf0);
    const int32_t par = src.parent[inner0 + k];
    dst.parent[k] = par < 0 ? par : par - inner0;
    for (int c = 0; c < 6; c++) dst.boxes[6 * (size_t)k + c] = src.boxes[6 * ((size_t)inner0 + k) + c];
  }
  if (k < n) {
    dst.geom[k] = src.geom[(size_t)leaf0 + k];
    dst.colour[k] = src.colour[(size_t)leaf0 + k];
    dst.morton[k] = src.morton[(size_t)leaf0 + k];
    dst.perm[k] = src.perm[(size_t)leaf0 + k] - leaf0;
  }
}

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace

size_t device_bvh_bytes(int64_t n_leaves, int32_t scenes, bool tables) {
  const size_t ni = (size_t)(n_leaves - scenes), nl = (size_t)n_leaves;
  size_t b = 0;
  b += 2 * align_up(ni * 64);       // nodes, nodes_soa
  b += 2 * align_up(nl * 16);       // geom, colour
  b += 2 * align_up(nl * 4);        // morton, perm
  b += 3 * align_up(ni * 4);        // left, right, parent
  b += align_up(ni * 24);           // boxes
  if (tables)                       // results, cameras, scene offsets
    b += align_up((size_t)scenes * sizeof(BvhBuildResult)) + align_up((size_t)scenes * 48) + align_up(((size_t)scenes + 1) * 4);
  return b;
}

void carve_device_bvh(unsigned char *block, int64_t n_leaves, DeviceBvh &out, int32_t scenes, bool tables) {
  const size_t ni = (size_t)(n_leaves - scenes), n = (size_t)n_leaves;
  unsigned char *p = block;
  auto carve = [&](size_t bytes) { unsigned char *r = p; p += align_up(bytes); return r; };
  out.block = block;
  out.block_bytes = device_bvh_bytes(n_leaves, scenes, tables);
  out.nodes = (float4 *)carve(ni * 64);
  out.nodes_soa = (float4 *)carve(ni * 64);
  out.geom = (float4 *)carve(n * 16);
  out.colour = (float4 *)carve(n * 16);
  out.morton = (uint32_t *)carve(n * 4);
  out.perm = (int32_t *)carve(n * 4);
  out.left = (int32_t *)carve(ni * 4);
  out.right = (int32_t *)carve(ni * 4);
  out.parent = (int32_t *)carve(ni * 4);
  out.boxes = (float *)carve(ni * 24);
  if (tables) {
    out.results = (BvhBuildResult *)carve((size_t)scenes * sizeof(BvhBuildResult));
    out.cams = (float *)carve((size_t)scenes * 48);
    out.scene_off = (int32_t *)carve(((size_t)scenes + 1) * 4);
  }
  out.n = (int32_t)n;
}

cudaError_t build_bvh_device(const float *d_spheres, int32_t scenes, const int32_t *off_host, const int32_t *sweeps_host, DeviceBvh &out,
                             BvhBuildResult *d_result, cudaStream_t stream, int64_t *launches) {
  const int total = off_host[scenes], ni = total - scenes;
  const bool batch = scenes > 1;
  int32_t max_sweeps = 0;
  bool same_sweeps = true, same_counts = true;
  for (int32_t b = 0; b < scenes; b++) {
    max_sweeps = sweeps_host[b] > max_sweeps ? sweeps_host[b] : max_sweeps;
    same_sweeps = same_sweeps && sweeps_host[b] == sweeps_host[0];
    same_counts = same_counts && off_host[b + 1] - off_host[b] == off_host[1];
  }
  int key_bits = 32, scene_bits = 0;  // a batch sorts (scene, key) and (scene, depth): the scene takes bits(scenes - 1)
  while (batch && ((int64_t)1 << scene_bits) < scenes) scene_bits++;
  key_bits += scene_bits;
  cudaError_t e;
  // ---- persistent outputs: one block, carved
  unsigned char *blk = nullptr;
  const bool tables = d_result == nullptr;  // a scene batch: the results go to its own table
  if ((e = cudaMallocAsync(&blk, device_bvh_bytes(total, scenes, tables), stream)) != cudaSuccess) return e;
  carve_device_bvh(blk, total, out, scenes, tables);
  if (tables) d_result = out.results;
  unsigned char *p = nullptr;
  auto carve = [&](size_t bytes) { unsigned char *r = p; p += align_up(bytes); return r; };

  // ---- scratch: one block, freed (stream-ordered) at the end
  size_t sort_tmp = 0, sort_tmp2 = 0;
  if (batch) {
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr,
                                    (int32_t *)nullptr, total, 0, key_bits, stream);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp2, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr,
                                    (int32_t *)nullptr, ni, 0, 8 + scene_bits, stream);
  } else {
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                    (int32_t *)nullptr, total, 0, 32, stream);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp2, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                    (int32_t *)nullptr, ni, 0, 8, stream);
  }
  const size_t cub_bytes = sort_tmp > sort_tmp2 ? sort_tmp : sort_tmp2;
  const size_t kw = batch ? 8 : 4;  // bytes of a sort key
  const size_t scratch_bytes = 3 * align_up((size_t)total * 4) /* cx cy cz */ + 2 * align_up((size_t)total * kw) /* key, sorted key (batch) */ +
                               align_up((size_t)total * 4) /* idx */ + align_up((size_t)ni * 24) /* boxes ping-pong */ +
                               3 * align_up((size_t)ni * 4) /* ids order newidx */ + 2 * align_up((size_t)ni * kw) /* depth, depth sorted */ +
                               align_up((size_t)scenes * 24) /* min/max */ + align_up((size_t)scenes * 8) /* depth, stale */ + align_up(cub_bytes) +
                               (batch ? align_up((size_t)ni * 4) /* node scenes */ + align_up((size_t)scenes * 4) /* sweeps */ : 0);
  unsigned char *scratch = nullptr;
  if ((e = cudaMallocAsync(&scratch, scratch_bytes, stream)) != cudaSuccess) return e;
  p = scratch;
  float *cx = (float *)carve((size_t)total * 4), *cy = (float *)carve((size_t)total * 4), *cz = (float *)carve((size_t)total * 4);
  void *key = carve((size_t)total * kw), *key_sorted = carve((size_t)total * kw);
  int32_t *idx = (int32_t *)carve((size_t)total * 4);
  float *boxes_b = (float *)carve((size_t)ni * 24);
  void *depth = carve((size_t)ni * kw), *depth_sorted = carve((size_t)ni * kw);
  int32_t *node_id = (int32_t *)carve((size_t)ni * 4);
  int32_t *order = (int32_t *)carve((size_t)ni * 4);
  int32_t *newidx = (int32_t *)carve((size_t)ni * 4);
  int *minmax = (int *)carve((size_t)scenes * 24);  // [scenes][6] min/max as ordered ints
  int *result = (int *)carve((size_t)scenes * 8);   // [scenes][2] max depth, stale
  void *cub_tmp = carve(cub_bytes);
  int32_t *node_scene = batch ? (int32_t *)carve((size_t)ni * 4) : nullptr;  // [ni] scene of every inner node
  int32_t *d_sweeps = batch && !same_sweeps ? (int32_t *)carve((size_t)scenes * 4) : nullptr;  // [scenes] refit sweeps
  // the offsets (a batch's block keeps them for the render kernels) and the sweep counts; the caller keeps the host
  // tables alive until the stream reaches these copies
  const int32_t *off = tables ? out.scene_off : nullptr;
  const Scenes S{off, scenes, same_counts ? off_host[1] : 0};
  if (tables) e = cudaMemcpyAsync(out.scene_off, off_host, ((size_t)scenes + 1) * 4, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess && d_sweeps) e = cudaMemcpyAsync(d_sweeps, sweeps_host, (size_t)scenes * 4, cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) { cudaFreeAsync(scratch, stream); return e; }

  // ---- bvh.fut:31-41
  init_build_kernel<<<blocks_for(scenes), kThreads, 0, stream>>>(minmax, result, scenes);
  const int64_t steps = (total + 31) / 32;                         // 32-sphere steps of centres_minmax_kernel
  const int64_t warps_max = 1056 * (kThreads / 32);                // 132 SMs x 8 blocks of 8 warps
  const int per_warp = (int)(32 * ((steps + warps_max - 1) / warps_max));
  const int64_t warps = (total + per_warp - 1) / per_warp;
  centres_minmax_kernel<<<(unsigned)((warps + kThreads / 32 - 1) / (kThreads / 32)), kThreads, 0, stream>>>(d_spheres, S, total,
                                                                                                               per_warp, cx, cy, cz, minmax);
  morton_kernel<<<blocks_for(total), kThreads, 0, stream>>>(cx, cy, cz, total, S, minmax, (uint32_t *)key,
                                                            batch ? (uint64_t *)key : nullptr, idx);
  // ---- bvh.fut:43 stable sort by the 32-bit key (a batch: by (scene, key))
  if (batch) {
    cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, (uint64_t *)key, (uint64_t *)key_sorted, idx, out.perm, total, 0, key_bits, stream);
    low_keys_kernel<<<blocks_for(total), kThreads, 0, stream>>>((const uint64_t *)key_sorted, total, out.morton);
  } else {
    cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, (uint32_t *)key, out.morton, idx, out.perm, total, 0, 32, stream);
  }
  // ---- radixtree.fut
  cudaMemsetAsync(out.parent, 0xff, (size_t)ni * 4, stream);
  karras_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.morton, S, total, out.left, out.right, out.parent, node_scene);
  // ---- bvh.fut:44-58 fixed number of Jacobi sweeps from zero boxes, each scene its own number (the largest runs, the
  // others' boxes are copied through the sweeps they do not run); the last sweep must land in out.boxes
  float *src = (max_sweeps % 2 == 0) ? out.boxes : boxes_b, *dst = (max_sweeps % 2 == 0) ? boxes_b : out.boxes;
  cudaMemsetAsync(src, 0, (size_t)ni * 24, stream);
  for (int s = 0; s < max_sweeps; s++) {
    refit_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(src, dst, out.left, out.right, d_spheres, out.perm, ni,
                                                          same_sweeps ? nullptr : d_sweeps, node_scene, s);
    float *t = src; src = dst; dst = t;
  }
  // (src now points at the final boxes == out.boxes)
  // ---- layout: order nodes by (depth, Karras index) (a batch: by (scene, depth, Karras index)), pack
  depth_stale_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.boxes, out.left, out.right, out.parent, d_spheres, out.perm, ni, node_scene,
                                                               (uint32_t *)depth, batch ? (uint64_t *)depth : nullptr, node_id, result);
  if (batch)
    cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp2, (uint64_t *)depth, (uint64_t *)depth_sorted, node_id, order, ni, 0, 8 + scene_bits, stream);
  else
    cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp2, (uint32_t *)depth, (uint32_t *)depth_sorted, node_id, order, ni, 0, 8, stream);
  invert_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(order, ni, newidx);
  pack_nodes_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.boxes, out.left, out.right, order, newidx, ni, out.nodes, out.nodes_soa);
  pack_spheres_kernel<<<blocks_for(total), kThreads, 0, stream>>>(d_spheres, out.perm, total, out.geom, out.colour);
  finish_kernel<<<blocks_for(scenes), kThreads, 0, stream>>>(out.boxes, result, S, d_result);
  if (launches) *launches += 10 + (batch ? 1 : 0) + max_sweeps + 2 /* cub passes are counted as one each */;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  return cudaFreeAsync(scratch, stream);
}

cudaError_t gather_spheres_device(const DeviceBvh &bvh, int64_t n, float *d_out, cudaStream_t stream, int64_t *launches) {
  gather_spheres_kernel<<<blocks_for(n), kThreads, 0, stream>>>(bvh.geom, bvh.colour, bvh.perm, n, d_out);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

cudaError_t extract_scene_device(const DeviceBvh &batch, int32_t s, int64_t off_s, int64_t n, DeviceBvh &out, cudaStream_t stream,
                                 int64_t *launches) {
  cudaError_t e;
  unsigned char *blk = nullptr;
  if ((e = cudaMallocAsync(&blk, device_bvh_bytes(n), stream)) != cudaSuccess) return e;
  carve_device_bvh(blk, n, out);
  extract_scene_kernel<<<blocks_for(n), kThreads, 0, stream>>>(batch, s, (int32_t)off_s, (int)n, out);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace rayb200
