// TEST INFRASTRUCTURE, NOT PRODUCT CODE: the CPU oracle of the occlusion query (include/ray_b200.h
// ray_b200_trace_occluded).
//
// The ray-query oracle (tests/ray_query_oracle.cpp, which includes oracle/oracle.cpp) is compiled into this translation
// unit unchanged, so every oracle_* entry of both exists here too and operates on this library's own handles.  On top of
// it: the reference's stackless bvh_fold walk folded with "some reached leaf accepts its sphere in (t_min, t_max)".
// tests/occlusion_oracle.py compiles it with oracle/Makefile's flags (strict f32: no FMA contraction, no -march, no
// fast-math).
#include "ray_query_oracle.cpp"

namespace {

// bvh.fut:61-84 bvh_fold inlined literally, as objs_hit_leaf walks it (boxes against (t_min, t_max), ray.fut:77), with
// the fold operator "acc or sphere_hit L[i] r t_min t_max" (ray.fut:32-51): some reached leaf accepts in the interval.
// The OR short-circuits the sphere test once acc is set; the walk itself is not cut short.
bool objs_occluded(const Bvh &bvh, const Ray &r, float t_min, float t_max) {
  bool acc = false;
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
      acc = acc || sphere_hit(bvh.L[child.idx], r, t_min, t_max, &h);
      prev = child;
    }
  }
  return acc;
}

}  // namespace

extern "C" {

// Occlusion per ray of rays (n x 6: origin.xyz, dir.xyz): out[i] = 1 if some leaf the walk reaches accepts its sphere
// in (t_min, t_max), else 0.
int oracle_trace_occluded(void *pv, const float *rays, int64_t n, float t_min, float t_max, uint8_t *out, int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays + 6 * i;
      out[i] = objs_occluded(p->objs, Ray{{q[0], q[1], q[2]}, {q[3], q[4], q[5]}}, t_min, t_max) ? 1 : 0;
    }
  });
  return 0;
}

}  // extern "C"
