// TEST INFRASTRUCTURE, NOT PRODUCT CODE: the CPU oracle of the ray queries whose rays carry their own interval
// (include/ray_b200.h struct ray_b200_ray, ray_b200_trace_*_ranged).
//
// The ray-query oracle (tests/ray_query_oracle.cpp, which compiles oracle/oracle.cpp unchanged) is included below
// unchanged, so every oracle_* entry of it exists here too and operates on this library's own handles.  On top of it: the
// three one-segment queries per ray, each ray with its own interval, through the same walk (objs_hit_leaf,
// objs_occluded, objs_accepted); there is no second walk.  tests/ray_interval_oracle.py compiles it with the ray-query
// oracle's flags (strict f32: no FMA contraction, no -march, no fast-math).
#include "ray_query_oracle.cpp"

namespace {

// The empty record: t = -1, sphere = -1, p = normal = 0.
void empty_record(float *o) {
  const int32_t none = -1;
  o[0] = -1.0f; memcpy(o + 1, &none, 4);
  for (int c = 2; c < 8; c++) o[c] = 0.0f;
}

// struct ray_b200_hit of a hit h on leaf `leaf`: t, bits(perm[leaf]), p.xyz, normal.xyz.
void write_record(const Prepared *p, const Hit &h, int32_t leaf, float *o) {
  const int32_t sphere = p->objs.perm[(size_t)leaf];
  o[0] = h.t; memcpy(o + 1, &sphere, 4);
  o[2] = h.p.x; o[3] = h.p.y; o[4] = h.p.z; o[5] = h.normal.x; o[6] = h.normal.y; o[7] = h.normal.z;
}

// A ray of struct ray_b200_ray (origin, t_min, direction, t_max), and whether its interval is one the per-call entry
// points accept: t_min finite and >= 0 (-0.0 included), t_max finite.  That rule is the library's contract for rays that
// carry their own interval, not the reference's: objs_hit would walk with a negative t_min.  An invalid ray gets the
// empty answer without a walk.
Ray ranged_ray(const float *q, bool *valid) {
  *valid = std::isfinite(q[3]) && q[3] >= 0.0f && std::isfinite(q[7]);
  return Ray{{q[0], q[1], q[2]}, {q[4], q[5], q[6]}};
}

}  // namespace

extern "C" {

// objs_hit objs r t_min t_max per ray of rays8 (n x 8), each with its own interval: out8 per ray = struct ray_b200_hit as
// oracle_trace_hits writes it.
int oracle_trace_hits_ranged(void *pv, const float *rays8, int64_t n, float *out8, int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays8 + 8 * i;
      float *o = out8 + 8 * i;
      bool valid;
      const Ray r = ranged_ray(q, &valid);
      Hit h;
      int32_t leaf = -1;
      if (valid && objs_hit_leaf(p->objs, r, q[3], q[7], &h, &leaf)) write_record(p, h, leaf, o);
      else empty_record(o);
    }
  });
  return 0;
}

// Occlusion per ray of rays8, each with its own interval: out[i] = 1 if some leaf the walk reaches accepts its sphere in
// (t_min, t_max), else 0.
int oracle_trace_occluded_ranged(void *pv, const float *rays8, int64_t n, uint8_t *out, int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays8 + 8 * i;
      bool valid;
      const Ray r = ranged_ray(q, &valid);
      out[i] = valid && objs_occluded(p->objs, r, q[3], q[7]) ? 1 : 0;
    }
  });
  return 0;
}

// Multi-hit per ray of rays8, each with its own interval: records and counts as oracle_trace_multi_hits writes them.
int oracle_trace_multi_hits_ranged(void *pv, const float *rays8, int64_t n, int32_t k, float *out8, int32_t *counts,
                                   int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0 || k < 1) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays8 + 8 * i;
      float *o = out8 + 8 * (size_t)i * (size_t)k;
      bool valid;
      const Ray r = ranged_ray(q, &valid);
      std::vector<Accepted> acc;
      if (valid) acc = objs_accepted(p->objs, r, q[3], q[7]);
      std::stable_sort(acc.begin(), acc.end(), [](const Accepted &a, const Accepted &b) {
        return a.t < b.t || (a.t == b.t && a.leaf < b.leaf);
      });
      for (int32_t j = 0; j < k; j++) {
        if ((size_t)j < acc.size()) write_record(p, acc[j].h, acc[j].leaf, o + 8 * (size_t)j);
        else empty_record(o + 8 * (size_t)j);
      }
      if (counts) counts[i] = (int32_t)acc.size();
    }
  });
  return 0;
}

}  // extern "C"
