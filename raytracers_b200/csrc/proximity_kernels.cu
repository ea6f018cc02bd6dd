// Proximity queries (include/ray_b200.h "proximity queries", DESIGN.md §5d): the spheres within a radius of each query
// point, nearest first.  One thread per ball walks the BVH2C records (scene_host.h) depth first, left child first, with
// a ball-box test that is conservative by a proved margin, and tests every sphere it reaches exactly.  This file shares
// no code with the render kernels: their hot loop stays as bench.py measures it.
//
// Scenes whose stored boxes are stale (the fixed-sweep refit stopped before its fixpoint) are walked over complete
// boxes that refit_complete_boxes builds first: a parent-pointer scatter, then a bottom-up pass in which the second
// thread to reach a record joins its two children (Karras' atomic-flag refit).
#include <cfloat>

#include "proximity.h"
#include "render_params.h"

namespace rayb200 {

namespace prox {  // named, so that the kernels keep stable names in profiles

constexpr int kThreads = 128;

// ---------------------------------------------------------------------------------------------- complete boxes

// par[j] = (k << 1) | side for the record k whose child `side` is inner record j; lpar[i] the same for leaf i
__global__ void prox_parents_kernel(const float4 *__restrict__ nodes, int n_inner, int32_t *__restrict__ par,
                                    int32_t *__restrict__ lpar) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_inner) return;
  const int ptr[2] = {__float_as_int(nodes[4 * (size_t)k].w), __float_as_int(nodes[4 * (size_t)k + 1].w)};
  for (int side = 0; side < 2; side++) {
    if (ptr[side] >= 0) par[ptr[side]] = k << 1 | side;
    else lpar[~ptr[side]] = k << 1 | side;
  }
}

// One thread per leaf climbs from the leaf's record to the root.  At each record the first of the two arriving threads
// stops; the second joins the record's two children (a leaf child's sphere box, an inner child's box as its own thread
// wrote it into this record) and writes the result into the parent record's slot for this record.  Every inner child
// slot is written exactly once, by the thread that completes the child; a root's own box goes nowhere.
__global__ void prox_refit_kernel(float4 *__restrict__ out, const float4 *__restrict__ geom, const int32_t *__restrict__ par,
                                  const int32_t *__restrict__ lpar, int32_t *__restrict__ arrived, int n_leaves) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_leaves) return;
  int q = lpar[i] >> 1;
  for (;;) {
    __threadfence();                                   // this thread's slot write before its arrival
    if (atomicAdd(arrived + q, 1) == 0) return;        // the sibling subtree is not complete yet
    __threadfence();                                   // the sibling's slot write before the reads below
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    const int ptrs[2] = {__float_as_int(__ldcg(&out[4 * (size_t)q].w)), __float_as_int(__ldcg(&out[4 * (size_t)q + 1].w))};
    for (int side = 0; side < 2; side++) {
      const float4 a = __ldcg(out + 4 * (size_t)q + 2 * side), b = __ldcg(out + 4 * (size_t)q + 2 * side + 1);
      const int ptr = ptrs[side];   // both child pointers live in q0.w and q1.w
      float c[6];
      if (ptr < 0) {  // sphere box, as the build's sphere_aabb computes it
        const float4 g = geom[~ptr];
        c[0] = g.x - g.w; c[1] = g.y - g.w; c[2] = g.z - g.w;
        c[3] = g.x + g.w; c[4] = g.y + g.w; c[5] = g.z + g.w;
      } else {
        c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = b.x; c[4] = b.y; c[5] = b.z;
      }
      for (int d = 0; d < 3; d++) { lo[d] = fminf(lo[d], c[d]); hi[d] = fmaxf(hi[d], c[3 + d]); }
    }
    const int up = par[q];
    if (up < 0) return;                                // a root
    float *slot = reinterpret_cast<float *>(out + 4 * (size_t)(up >> 1) + 2 * (up & 1));
    for (int d = 0; d < 3; d++) { __stcg(slot + d, lo[d]); __stcg(slot + 4 + d, hi[d]); }  // .w holds child pointers
    q = up >> 1;
  }
}

// ---------------------------------------------------------------------------------------------- the query

// The ball-box test, in two parts that both query kernels use: the bound G, a lower bound of the squared distance from c
// to the box rounded down, and the threshold, an upper bound of (r + 2^-20 (r + M) + FLT_MIN)^2 rounded up, where M is
// the box's largest coordinate magnitude.  A box may hold a sphere within the ball (c, r) when !(G > threshold).
// DESIGN.md §5d proves that every sphere with d <= r passes every complete box above it.  NaN coordinates pass (fmaxf
// drops them, and a NaN bound compares false); a box with an infinite coordinate gets an infinite threshold unless c is
// infinitely far from it, and r = +inf gives an infinite threshold.
__device__ __forceinline__ float box_gap2(float cx, float cy, float cz, const float4 lo, const float4 hi) {
  const float gx = fmaxf(fmaxf(__fsub_rd(lo.x, cx), __fsub_rd(cx, hi.x)), 0.0f);
  const float gy = fmaxf(fmaxf(__fsub_rd(lo.y, cy), __fsub_rd(cy, hi.y)), 0.0f);
  const float gz = fmaxf(fmaxf(__fsub_rd(lo.z, cz), __fsub_rd(cz, hi.z)), 0.0f);
  return __fadd_rd(__fadd_rd(__fmul_rd(gx, gx), __fmul_rd(gy, gy)), __fmul_rd(gz, gz));
}

__device__ __forceinline__ float box_mag(const float4 lo, const float4 hi) {
  return fmaxf(fmaxf(fmaxf(fabsf(lo.x), fabsf(lo.y)), fmaxf(fabsf(lo.z), fabsf(hi.x))), fmaxf(fabsf(hi.y), fabsf(hi.z)));
}

__device__ __forceinline__ float ball_reach2(float r, float m) {
  const float s = __fadd_ru(__fadd_ru(r, __fmul_ru(0x1p-20f, __fadd_ru(r, m))), FLT_MIN);
  return __fmul_ru(s, s);
}

__device__ __forceinline__ bool ball_meets_box(float cx, float cy, float cz, float r, const float4 lo, const float4 hi) {
  const float g2 = box_gap2(cx, cy, cz, lo, hi);
  return !(g2 > ball_reach2(r, box_mag(lo, hi)));
}

// (d, s) before (d2, s2): ascending distance, then ascending caller index.  kInfD: records may have d = +inf (a ball
// with no limit reports spheres whose d overflows), so the index compares unsigned and the unused record (+inf, -1)
// stays after every record.
template <bool kInfD = false>
__device__ __forceinline__ bool before(float d, int s, float d2, int s2) {
  return d < d2 || (d == d2 && (kInfD ? (unsigned)s < (unsigned)s2 : s < s2));
}

// The k best records of one ball.  KB = 0: none (count only); 1 and 8: in registers (the first k of KB); 64: in the
// ball's own output row, kept sorted there.  kth(): the k-th record once k are held (the nearest-sphere query's d_k).
template <int KB, bool kInfD = false>
struct Best {
  float d[KB];
  int s[KB];
  __device__ __forceinline__ void init(float2 *, int) {
#pragma unroll
    for (int j = 0; j < KB; j++) { d[j] = INFINITY; s[j] = -1; }
  }
  __device__ __forceinline__ void kth(float2 *, int k, int, float &dk, int &sk) const {
    // the last slot below k wins: predicated moves (an equality select becomes an indexed load from local memory)
#pragma unroll
    for (int j = 0; j < KB; j++) {
      if (j < k) { dk = d[j]; sk = s[j]; }
    }
  }
  __device__ __forceinline__ void insert(float2 *, int, int, float cd, int cs) {
#pragma unroll
    for (int j = 0; j < KB; j++) {
      if (before<kInfD>(cd, cs, d[j], s[j])) {
        const float td = d[j]; const int ts = s[j];
        d[j] = cd; s[j] = cs; cd = td; cs = ts;
      }
    }
  }
  __device__ __forceinline__ void store(float2 *row, int k) {
#pragma unroll
    for (int j = 0; j < KB; j++) {
      if (j < k) {
        float *e = reinterpret_cast<float *>(row + j);
        e[0] = d[j];
        e[1] = __int_as_float(s[j]);
      }
    }
  }
};

template <>
struct Best<0> {
  __device__ __forceinline__ void init(float2 *, int) {}
  __device__ __forceinline__ void insert(float2 *, int, int, float, int) {}
  __device__ __forceinline__ void store(float2 *, int) {}
};

// The row's records are compared with each other only, never with an unused one, so one order serves both queries
template <bool kInfD>
struct Best<64, kInfD> {
  // the row is 4-byte aligned (struct ray_b200_near): word loads and stores
  __device__ __forceinline__ static float &dist(float2 *row, int j) { return reinterpret_cast<float *>(row)[2 * j]; }
  __device__ __forceinline__ static float &idx(float2 *row, int j) { return reinterpret_cast<float *>(row)[2 * j + 1]; }
  __device__ __forceinline__ void init(float2 *row, int k) {
    for (int j = 0; j < k; j++) { dist(row, j) = INFINITY; idx(row, j) = __int_as_float(-1); }
  }
  // `have`: the records held, this one included
  __device__ __forceinline__ void kth(float2 *row, int k, int have, float &dk, int &sk) const {
    if (have >= k) { dk = dist(row, k - 1); sk = __float_as_int(idx(row, k - 1)); }
  }
  // `have`: the records so far (the count before this sphere), of which min(have, k) are in the row
  __device__ __forceinline__ void insert(float2 *row, int k, int have, float cd, int cs) {
    int pos;
    if (have < k) {
      pos = have;
    } else {
      if (!before(cd, cs, dist(row, k - 1), __float_as_int(idx(row, k - 1)))) return;
      pos = k - 1;
    }
    while (pos > 0 && before(cd, cs, dist(row, pos - 1), __float_as_int(idx(row, pos - 1)))) {
      dist(row, pos) = dist(row, pos - 1);
      idx(row, pos) = idx(row, pos - 1);
      pos--;
    }
    dist(row, pos) = cd;
    idx(row, pos) = __int_as_float(cs);
  }
  __device__ __forceinline__ void store(float2 *, int) {}
};

template <int KB>
__global__ void __launch_bounds__(kThreads) prox_query_kernel(const ProximityQuery Q) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q.n) return;
  const float *ball = Q.balls + 4 * i;
  const float cx = __ldg(ball), cy = __ldg(ball + 1), cz = __ldg(ball + 2), r = __ldg(ball + 3);
  int root = 0, base = 0;
  if (Q.scene_off) {
    const int b = (int)(i / Q.balls_per_scene);
    base = __ldg(Q.scene_off + b);
    root = base - b;
  }
  const int k = Q.k;
  float2 *row = KB ? reinterpret_cast<float2 *>(Q.near) + i * k : nullptr;
  Best<KB> best;
  best.init(row, k);
  int count = 0;
  // an invalid ball gets the empty answer (include/ray_b200.h)
  if (isfinite(cx) && isfinite(cy) && isfinite(cz) && isfinite(r) && r >= 0.0f) {
    int stack[kStackSize];
    int sp = 0, cur = root;
    for (;;) {
      const float4 *rec = Q.nodes + 4 * (size_t)cur;
      const float4 q0 = __ldg(rec), q1 = __ldg(rec + 1), q2 = __ldg(rec + 2), q3 = __ldg(rec + 3);
      const int lptr = __float_as_int(q0.w), rptr = __float_as_int(q1.w);
      // leaf children are tested as they are reached; their stored boxes always pass
#pragma unroll
      for (int side = 0; side < 2; side++) {
        const int ptr = side == 0 ? lptr : rptr;
        if (ptr >= 0) continue;
        const float4 g = __ldg(Q.geom + ~ptr);
        // a sphere with a non-finite centre or radius, or a negative or NaN radius, is never reported (-0.0 is a point)
        if (!(isfinite(g.x) && isfinite(g.y) && isfinite(g.z) && isfinite(g.w) && g.w >= 0.0f)) continue;
        const float dx = __fsub_rn(g.x, cx), dy = __fsub_rn(g.y, cy), dz = __fsub_rn(g.z, cz);
        const float d = __fsub_rn(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), g.w);
        if (d <= r) {
          best.insert(row, k, count, d, __ldg(Q.perm + ~ptr) - base);
          count++;
        }
      }
      const bool tl = lptr >= 0 && ball_meets_box(cx, cy, cz, r, q0, q1);
      const bool tr = rptr >= 0 && ball_meets_box(cx, cy, cz, r, q2, q3);
      if (tl && tr) stack[sp++] = rptr;
      if (tl || tr) {
        cur = tl ? lptr : rptr;
      } else {
        if (sp == 0) break;
        cur = stack[--sp];
      }
    }
  }
  best.store(row, k);
  if (Q.counts) Q.counts[i] = count;
}

// The k nearest spheres within a ball whose r may be +inf (include/ray_b200.h "nearest-sphere queries", DESIGN.md §5e).
// The walk prunes with R = max(0, min(r, d_k)), d_k the k-th best d so far (+inf while fewer than k are held): R only
// shrinks, every final record has d <= R throughout, so by §5d it passes every complete box above it.  Each record's
// two children are ordered by their bounds G, the nearer one is walked first and the other is pushed with G and its box's
// magnitude M, so that a pop tests it again against the R of that moment and drops it without loading its record.
template <int KB>
__global__ void __launch_bounds__(kThreads) prox_nearest_kernel(const ProximityQuery Q) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q.n) return;
  const float *ball = Q.balls + 4 * i;
  const float cx = __ldg(ball), cy = __ldg(ball + 1), cz = __ldg(ball + 2), r = __ldg(ball + 3);
  int root = 0, base = 0;
  if (Q.scene_off) {
    const int b = (int)(i / Q.balls_per_scene);
    base = __ldg(Q.scene_off + b);
    root = base - b;
  }
  const int k = Q.k;
  float2 *row = reinterpret_cast<float2 *>(Q.near) + i * k;
  Best<KB, true> best;
  best.init(row, k);
  // an invalid ball gets the empty answer: r = +inf is valid, r NaN or negative is not (include/ray_b200.h)
  if (isfinite(cx) && isfinite(cy) && isfinite(cz) && r >= 0.0f) {
    float dk = INFINITY, R = r;     // d_k and R; the k-th record's caller index is sk
    int sk = -1, have = 0;
    int stack[kStackSize];
    float stack_g[kStackSize], stack_m[kStackSize];
    int sp = 0, cur = root;
    for (;;) {
      const float4 *rec = Q.nodes + 4 * (size_t)cur;
      const float4 q0 = __ldg(rec), q1 = __ldg(rec + 1), q2 = __ldg(rec + 2), q3 = __ldg(rec + 3);
      const int lptr = __float_as_int(q0.w), rptr = __float_as_int(q1.w);
#pragma unroll
      for (int side = 0; side < 2; side++) {
        const int ptr = side == 0 ? lptr : rptr;
        if (ptr >= 0) continue;
        const float4 g = __ldg(Q.geom + ~ptr);
        if (!(isfinite(g.x) && isfinite(g.y) && isfinite(g.z) && isfinite(g.w) && g.w >= 0.0f)) continue;
        const float dx = __fsub_rn(g.x, cx), dy = __fsub_rn(g.y, cy), dz = __fsub_rn(g.z, cz);
        const float d = __fsub_rn(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), g.w);
        // d <= R is needed to be within r and before the k-th record; the caller index breaks a tie at d_k
        if (!(d <= R)) continue;
        const int s = __ldg(Q.perm + ~ptr) - base;
        if (!before<true>(d, s, dk, sk)) continue;
        best.insert(row, k, have, d, s);
        have++;
        best.kth(row, k, have, dk, sk);
        R = fmaxf(fminf(r, dk), 0.0f);
      }
      float gl = 0.0f, gr = 0.0f, ml = 0.0f, mr = 0.0f;
      bool tl = false, tr = false;
      if (lptr >= 0) {
        gl = box_gap2(cx, cy, cz, q0, q1);
        ml = box_mag(q0, q1);
        tl = !(gl > ball_reach2(R, ml));
      }
      if (rptr >= 0) {
        gr = box_gap2(cx, cy, cz, q2, q3);
        mr = box_mag(q2, q3);
        tr = !(gr > ball_reach2(R, mr));
      }
      if (tl && tr) {
        const bool left_first = !(gr < gl);   // ties (and a NaN bound) go left first
        stack[sp] = left_first ? rptr : lptr;
        stack_g[sp] = left_first ? gr : gl;
        stack_m[sp] = left_first ? mr : ml;
        sp++;
        cur = left_first ? lptr : rptr;
      } else if (tl || tr) {
        cur = tl ? lptr : rptr;
      } else {
        // pop the next entry that still passes against the current R
        cur = -1;
        while (sp > 0) {
          sp--;
          if (!(stack_g[sp] > ball_reach2(R, stack_m[sp]))) { cur = stack[sp]; break; }
        }
        if (cur < 0) break;
      }
    }
  }
  best.store(row, k);
}

inline unsigned blocks_for(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace prox

using namespace prox;

size_t refit_scratch_bytes(int64_t n_inner, int64_t n_leaves) {
  return 2 * align_up((size_t)n_inner * sizeof(int32_t)) + align_up((size_t)n_leaves * sizeof(int32_t));
}

cudaError_t refit_complete_boxes(const float4 *nodes, const float4 *geom, int64_t n_inner, int64_t n_leaves, float4 *out,
                                 void *scratch, cudaStream_t stream, int64_t *launches) {
  unsigned char *s = static_cast<unsigned char *>(scratch);
  int32_t *par = reinterpret_cast<int32_t *>(s);
  int32_t *arrived = reinterpret_cast<int32_t *>(s + align_up((size_t)n_inner * sizeof(int32_t)));
  int32_t *lpar = reinterpret_cast<int32_t *>(s + 2 * align_up((size_t)n_inner * sizeof(int32_t)));
  cudaError_t e;
  if ((e = cudaMemcpyAsync(out, nodes, (size_t)n_inner * 4 * sizeof(float4), cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(par, 0xFF, (size_t)n_inner * sizeof(int32_t), stream)) != cudaSuccess) return e;   // roots: -1
  if ((e = cudaMemsetAsync(arrived, 0, (size_t)n_inner * sizeof(int32_t), stream)) != cudaSuccess) return e;
  prox_parents_kernel<<<blocks_for(n_inner), kThreads, 0, stream>>>(nodes, (int)n_inner, par, lpar);
  prox_refit_kernel<<<blocks_for(n_leaves), kThreads, 0, stream>>>(out, geom, par, lpar, arrived, (int)n_leaves);
  if (launches) *launches += 2;
  return cudaGetLastError();
}

cudaError_t launch_proximity(const ProximityQuery &Q, cudaStream_t stream, int64_t *launches) {
  const unsigned g = blocks_for(Q.n);
  if (Q.k == 0) prox_query_kernel<0><<<g, kThreads, 0, stream>>>(Q);
  else if (Q.k == 1) prox_query_kernel<1><<<g, kThreads, 0, stream>>>(Q);
  else if (Q.k <= 8) prox_query_kernel<8><<<g, kThreads, 0, stream>>>(Q);
  else prox_query_kernel<64><<<g, kThreads, 0, stream>>>(Q);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

cudaError_t launch_nearest(const ProximityQuery &Q, cudaStream_t stream, int64_t *launches) {
  const unsigned g = blocks_for(Q.n);
  if (Q.k == 1) prox_nearest_kernel<1><<<g, kThreads, 0, stream>>>(Q);
  else if (Q.k <= 8) prox_nearest_kernel<8><<<g, kThreads, 0, stream>>>(Q);
  else prox_nearest_kernel<64><<<g, kThreads, 0, stream>>>(Q);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace rayb200
