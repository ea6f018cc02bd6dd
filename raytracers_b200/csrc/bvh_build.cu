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

// bvh.fut:31-37: centre of every sphere box (prim.fut:47-50) and the six min/max reductions over them.
__global__ void centres_minmax_kernel(const float *__restrict__ spheres, int n, float *__restrict__ cx,
                                      float *__restrict__ cy, float *__restrict__ cz, int *__restrict__ minmax /* [6] ordered ints */) {
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const SphereBox b = sphere_box(spheres + 7 * (size_t)k);
    const float c[3] = {b.lo[0] + 0.5f * (b.hi[0] - b.lo[0]), b.lo[1] + 0.5f * (b.hi[1] - b.lo[1]),
                        b.lo[2] + 0.5f * (b.hi[2] - b.lo[2])};
    cx[k] = c[0]; cy[k] = c[1]; cz[k] = c[2];
    for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], c[a]); hi[a] = fmaxf(hi[a], c[a]); }
  }
  for (int a = 0; a < 3; a++) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_down_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_down_sync(0xffffffffu, hi[a], o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(minmax + a, float_to_ordered(lo[a]));
      atomicMax(minmax + 3 + a, float_to_ordered(hi[a]));
    }
  }
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

// bvh.fut:38-41 + morton_3D (bvh.fut:15-22)
__global__ void morton_kernel(const float *__restrict__ cx, const float *__restrict__ cy, const float *__restrict__ cz, int n,
                              const int *__restrict__ minmax, uint32_t *__restrict__ key, int32_t *__restrict__ idx) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float lo[3] = {ordered_to_float(minmax[0]), ordered_to_float(minmax[1]), ordered_to_float(minmax[2])};
  const float hi[3] = {ordered_to_float(minmax[3]), ordered_to_float(minmax[4]), ordered_to_float(minmax[5])};
  const uint32_t qx = quantise10((cx[k] - lo[0]) / (hi[0] - lo[0]));
  const uint32_t qy = quantise10((cy[k] - lo[1]) / (hi[1] - lo[1]));
  const uint32_t qz = quantise10((cz[k] - lo[2]) / (hi[2] - lo[2]));
  key[k] = spread10(qx) * 4u + spread10(qy) * 2u + spread10(qz);
  idx[k] = k;
}

// mk_radix_tree (radixtree.fut:11-72): one thread per inner node.
__global__ void karras_kernel(const uint32_t *__restrict__ M, int n, int32_t *__restrict__ left, int32_t *__restrict__ right,
                              int32_t *__restrict__ parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n - 1) return;
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
  const int l = (min(i, j) == gamma) ? ~gamma : gamma;           // :54-57
  const int r = (max(i, j) == gamma + 1) ? ~(gamma + 1) : gamma + 1;  // :59-62
  left[i] = l;
  right[i] = r;
  if (l >= 0) parent[l] = i;                                     // :66-70 (scatter; the root keeps -1)
  if (r >= 0) parent[r] = i;
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

// one Jacobi sweep of bvh.fut:52-58: new boxes from the OLD boxes of the children
__global__ void refit_kernel(const float *__restrict__ src, float *__restrict__ dst, const int32_t *__restrict__ left,
                             const int32_t *__restrict__ right, const float *__restrict__ spheres, const int32_t *__restrict__ perm,
                             int ni) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ni) return;
  float a[6], b[6];
  child_box(src, spheres, perm, left[k], a);
  child_box(src, spheres, perm, right[k], b);
  float *o = dst + 6 * (size_t)k;
  for (int c = 0; c < 3; c++) { o[c] = min_num(a[c], b[c]); o[3 + c] = max_num(a[3 + c], b[3 + c]); }  // enclosing, prim.fut:38-45
}

// diagnostics + layout keys: depth of every inner node (root = 0) and how many boxes are not the union of their children
__global__ void depth_stale_kernel(const float *__restrict__ boxes, const int32_t *__restrict__ left, const int32_t *__restrict__ right,
                                   const int32_t *__restrict__ parent, const float *__restrict__ spheres, const int32_t *__restrict__ perm,
                                   int ni, uint32_t *__restrict__ depth, int32_t *__restrict__ node_id, int *__restrict__ result /* [0]=max depth,[1]=stale */) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ni) return;
  int d = 0;
  for (int p = parent[k]; p >= 0; p = parent[p]) d++;
  depth[k] = (uint32_t)d;
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

__global__ void finish_kernel(const float *__restrict__ boxes, const int *__restrict__ result, BvhBuildResult *__restrict__ out) {
  for (int c = 0; c < 6; c++) out->root_box[c] = boxes[c];
  out->max_depth = result[0];
  out->stale_nodes = result[1];
}

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace

size_t device_bvh_bytes(int64_t n) {
  const size_t ni = (size_t)(n - 1);
  size_t b = 0;
  b += 2 * align_up(ni * 64);       // nodes, nodes_soa
  b += 2 * align_up((size_t)n * 16);  // geom, colour
  b += 2 * align_up((size_t)n * 4);   // morton, perm
  b += 3 * align_up(ni * 4);        // left, right, parent
  b += align_up(ni * 24);           // boxes
  return b;
}

void carve_device_bvh(unsigned char *block, int64_t n64, DeviceBvh &out) {
  const size_t n = (size_t)n64, ni = n - 1;
  unsigned char *p = block;
  auto carve = [&](size_t bytes) { unsigned char *r = p; p += align_up(bytes); return r; };
  out.block = block;
  out.block_bytes = device_bvh_bytes(n64);
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
  out.n = (int32_t)n;
}

cudaError_t build_bvh_device(const float *d_spheres, int64_t n64, int32_t refit_sweeps, DeviceBvh &out, BvhBuildResult *d_result,
                             cudaStream_t stream, int64_t *launches) {
  const int n = (int)n64, ni = n - 1;
  cudaError_t e;
  // ---- persistent outputs: one block, carved
  unsigned char *blk = nullptr;
  if ((e = cudaMallocAsync(&blk, device_bvh_bytes(n), stream)) != cudaSuccess) return e;
  carve_device_bvh(blk, n, out);
  unsigned char *p = nullptr;
  auto carve = [&](size_t bytes) { unsigned char *r = p; p += align_up(bytes); return r; };

  // ---- scratch: one block, freed (stream-ordered) at the end
  size_t sort_tmp = 0, sort_tmp2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                  (int32_t *)nullptr, n, 0, 32, stream);
  cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp2, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                  (int32_t *)nullptr, ni, 0, 8, stream);
  const size_t cub_bytes = sort_tmp > sort_tmp2 ? sort_tmp : sort_tmp2;
  const size_t scratch_bytes = 3 * align_up((size_t)n * 4) /* cx cy cz */ + 2 * align_up((size_t)n * 4) /* key idx */ +
                               align_up((size_t)ni * 24) /* boxes ping-pong */ + 4 * align_up((size_t)ni * 4) /* depth ids order newidx */ +
                               align_up((size_t)ni * 4) /* depth sorted */ + align_up(64) + align_up(cub_bytes);
  unsigned char *scratch = nullptr;
  if ((e = cudaMallocAsync(&scratch, scratch_bytes, stream)) != cudaSuccess) return e;
  p = scratch;
  float *cx = (float *)carve((size_t)n * 4), *cy = (float *)carve((size_t)n * 4), *cz = (float *)carve((size_t)n * 4);
  uint32_t *key = (uint32_t *)carve((size_t)n * 4);
  int32_t *idx = (int32_t *)carve((size_t)n * 4);
  float *boxes_b = (float *)carve((size_t)ni * 24);
  uint32_t *depth = (uint32_t *)carve((size_t)ni * 4);
  int32_t *node_id = (int32_t *)carve((size_t)ni * 4);
  int32_t *order = (int32_t *)carve((size_t)ni * 4);
  int32_t *newidx = (int32_t *)carve((size_t)ni * 4);
  uint32_t *depth_sorted = (uint32_t *)carve((size_t)ni * 4);
  int *small = (int *)carve(64);  // [0..5] min/max as ordered ints, [8] max depth, [9] stale
  void *cub_tmp = carve(cub_bytes);

  // ---- bvh.fut:31-41
  const int init[6] = {0x7fffffff, 0x7fffffff, 0x7fffffff, (int)0x80000000, (int)0x80000000, (int)0x80000000};
  // ordered-int identity elements: +inf-ish for min, -inf-ish for max (any real float beats them)
  cudaMemsetAsync(small, 0, 64, stream);
  cudaMemcpyAsync(small, init, sizeof init, cudaMemcpyHostToDevice, stream);
  unsigned rb = blocks_for(n);
  if (rb > 1056) rb = 1056;  // 132 SMs x 8: grid-stride reduction
  centres_minmax_kernel<<<rb, kThreads, 0, stream>>>(d_spheres, n, cx, cy, cz, small);
  morton_kernel<<<blocks_for(n), kThreads, 0, stream>>>(cx, cy, cz, n, small, key, idx);
  // ---- bvh.fut:43 stable sort by the 32-bit key
  cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, key, out.morton, idx, out.perm, n, 0, 32, stream);
  // ---- radixtree.fut
  cudaMemsetAsync(out.parent, 0xff, (size_t)ni * 4, stream);
  karras_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.morton, n, out.left, out.right, out.parent);
  // ---- bvh.fut:44-58 fixed number of Jacobi sweeps from zero boxes; the last sweep must land in out.boxes
  float *src = (refit_sweeps % 2 == 0) ? out.boxes : boxes_b, *dst = (refit_sweeps % 2 == 0) ? boxes_b : out.boxes;
  cudaMemsetAsync(src, 0, (size_t)ni * 24, stream);
  for (int s = 0; s < refit_sweeps; s++) {
    refit_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(src, dst, out.left, out.right, d_spheres, out.perm, ni);
    float *t = src; src = dst; dst = t;
  }
  // (src now points at the final boxes == out.boxes)
  // ---- layout: order nodes by (depth, Karras index), pack
  depth_stale_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.boxes, out.left, out.right, out.parent, d_spheres, out.perm, ni, depth,
                                                               node_id, small + 8);
  cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp2, depth, depth_sorted, node_id, order, ni, 0, 8, stream);
  invert_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(order, ni, newidx);
  pack_nodes_kernel<<<blocks_for(ni), kThreads, 0, stream>>>(out.boxes, out.left, out.right, order, newidx, ni, out.nodes, out.nodes_soa);
  pack_spheres_kernel<<<blocks_for(n), kThreads, 0, stream>>>(d_spheres, out.perm, n, out.geom, out.colour);
  finish_kernel<<<1, 1, 0, stream>>>(out.boxes, small + 8, d_result);
  if (launches) *launches += 9 + refit_sweeps + 2 /* cub passes are counted as one each */;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  return cudaFreeAsync(scratch, stream);
}

cudaError_t gather_spheres_device(const DeviceBvh &bvh, int64_t n, float *d_out, cudaStream_t stream, int64_t *launches) {
  gather_spheres_kernel<<<blocks_for(n), kThreads, 0, stream>>>(bvh.geom, bvh.colour, bvh.perm, n, d_out);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace rayb200
