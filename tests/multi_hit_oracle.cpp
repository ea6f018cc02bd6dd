// TEST INFRASTRUCTURE, NOT PRODUCT CODE: the CPU oracle of the multi-hit query (include/ray_b200.h
// ray_b200_trace_multi_hits).
//
// The ray-query oracle (tests/ray_query_oracle.cpp, which includes oracle/oracle.cpp) is compiled into this translation
// unit unchanged, so every oracle_* entry of both exists here too and operates on this library's own handles.  On top of
// it: the reference's stackless bvh_fold walk folded with "collect (t, i) when sphere_hit L[i] r t_min t_max accepts",
// then a stable sort by (t, i).  tests/multi_hit_oracle.py compiles it with oracle/Makefile's flags (strict f32: no FMA
// contraction, no -march, no fast-math).
#include "ray_query_oracle.cpp"

namespace {

struct Accepted { float t; int32_t leaf; Hit h; };

// bvh.fut:61-84 bvh_fold inlined literally, as objs_hit_leaf walks it (boxes against (t_min, t_max), ray.fut:77), with
// the fold operator "acc ++ [(t, i)] if sphere_hit L[i] r t_min t_max" (ray.fut:32-51): every reached leaf that accepts
// in the interval, in walk order.
std::vector<Accepted> objs_accepted(const Bvh &bvh, const Ray &r, float t_min, float t_max) {
  std::vector<Accepted> acc;
  int32_t cur = 0;
  Ptr prev = inner_ptr(-1);
  while (cur != -1) {                                                  // bvh.fut:64
    const Inner &node = bvh.I[cur];
    bool from_left = ptr_eq(prev, node.left);
    bool from_right = ptr_eq(prev, node.right);
    bool rec = false;
    Ptr child = {0, 0};
    if (from_left) { rec = true; child = node.right; }                 // bvh.fut:70-71
    else if (!from_right) {                                            // bvh.fut:73-76
      if (aabb_hit(node.aabb, r, t_min, t_max)) { rec = true; child = node.left; }
    }
    if (!rec) { prev = inner_ptr(cur); cur = node.parent; }            // bvh.fut:79-80
    else if (child.tag == 1) { prev = inner_ptr(cur); cur = child.idx; }  // bvh.fut:83
    else {                                                             // bvh.fut:84: op acc i L[i]
      Hit h;
      if (sphere_hit(bvh.L[child.idx], r, t_min, t_max, &h)) acc.push_back({h.t, child.idx, h});
      prev = child;
    }
  }
  return acc;
}

}  // namespace

extern "C" {

// Multi-hit per ray of rays (n x 6: origin.xyz, dir.xyz): the accepted leaves stable-sorted by (t, leaf), the first k as
// out8[i][j] = struct ray_b200_hit (t, bits(perm[leaf]), p.xyz, normal.xyz from sphere_hit's own Hit), the rest t = -1,
// sphere = -1, p = normal = 0; counts[i] = the number of accepted leaves (counts may be NULL).
int oracle_trace_multi_hits(void *pv, const float *rays, int64_t n, float t_min, float t_max, int32_t k, float *out8,
                            int32_t *counts, int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0 || k < 1) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays + 6 * i;
      std::vector<Accepted> acc = objs_accepted(p->objs, Ray{{q[0], q[1], q[2]}, {q[3], q[4], q[5]}}, t_min, t_max);
      std::stable_sort(acc.begin(), acc.end(), [](const Accepted &a, const Accepted &b) {
        return a.t < b.t || (a.t == b.t && a.leaf < b.leaf);
      });
      for (int32_t j = 0; j < k; j++) {
        float *o = out8 + 8 * ((size_t)i * (size_t)k + (size_t)j);
        if ((size_t)j < acc.size()) {
          const Hit &h = acc[j].h;
          const int32_t sphere = p->objs.perm[(size_t)acc[j].leaf];
          o[0] = h.t; memcpy(o + 1, &sphere, 4);
          o[2] = h.p.x; o[3] = h.p.y; o[4] = h.p.z; o[5] = h.normal.x; o[6] = h.normal.y; o[7] = h.normal.z;
        } else {
          const int32_t none = -1;
          o[0] = -1.0f; memcpy(o + 1, &none, 4);
          for (int c = 2; c < 8; c++) o[c] = 0.0f;
        }
      }
      if (counts) counts[i] = (int32_t)acc.size();
    }
  });
  return 0;
}

}  // extern "C"
