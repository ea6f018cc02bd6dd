// TEST INFRASTRUCTURE, NOT PRODUCT CODE: the CPU oracle of the ray queries (include/ray_b200.h "ray queries").
//
// The literal restatement of the reference in oracle/oracle.cpp is compiled into this translation unit unchanged (it is
// included below), so every oracle_* entry of liboracle.so exists here too and operates on this library's own handles.
// On top of it: the reference's stackless bvh_fold walk for caller-supplied rays and intervals, folded three ways:
// objs_hit (ray.fut:76-86) reporting the winning leaf, "some reached leaf accepts its sphere in (t_min, t_max)" (the
// occlusion query) and "every reached leaf that accepts" (the multi-hit query); the same three one-segment queries for
// rays that carry their own interval (struct ray_b200_ray, ray_b200_trace_*_ranged), through the same walk; ray_colour
// with any depth limit (ray.fut:126-148); and the camera rays of oracle_render.  tests/ray_query_oracle.py compiles it
// with oracle/Makefile's flags (strict f32: no FMA contraction, no -march, no fast-math).
#include "../oracle/oracle.cpp"

#include <functional>

namespace {

// bvh.fut:61-84 bvh_fold inlined literally, as oracle.cpp's objs_hit walks it, with the boxes tested against
// (t_min, t_max) (ray.fut:77, the original t range); op(i) is the fold operator "op acc i L[i]" of every reached leaf i.
template <class Op>
void bvh_fold(const Bvh &bvh, const Ray &r, float t_min, float t_max, Op &&op) {
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
      op(child.idx);
      prev = child;
    }
  }
}

// ray.fut:76-86 objs_hit, as oracle.cpp's objs_hit, plus acc_j: the winning leaf in Morton order (-1 = none).
bool objs_hit_leaf(const Bvh &bvh, const Ray &r, float t_min, float t_max, Hit *out, int32_t *leaf) {
  int32_t acc_j = -1;
  float acc_t = t_max;
  bvh_fold(bvh, r, t_min, t_max, [&](int32_t i) {
    Hit h;
    if (sphere_hit(bvh.L[i], r, scene_epsilon, acc_t, &h)) { acc_j = i; acc_t = h.t; }  // ray.fut:78-81
  });
  *leaf = acc_j;
  if (acc_j >= 0) return sphere_hit(bvh.L[acc_j], r, t_min, acc_t + 1.0f, out);   // ray.fut:83-85
  return false;
}

// The fold operator "acc or sphere_hit L[i] r t_min t_max" (ray.fut:32-51): some reached leaf accepts in the interval.
// The OR short-circuits the sphere test once acc is set; the walk itself is not cut short.
bool objs_occluded(const Bvh &bvh, const Ray &r, float t_min, float t_max) {
  bool acc = false;
  bvh_fold(bvh, r, t_min, t_max, [&](int32_t i) {
    Hit h;
    acc = acc || sphere_hit(bvh.L[i], r, t_min, t_max, &h);
  });
  return acc;
}

struct Accepted { float t; int32_t leaf; Hit h; };

// The fold operator "acc ++ [(t, i)] if sphere_hit L[i] r t_min t_max" (ray.fut:32-51): every reached leaf that
// accepts in the interval, in walk order.
std::vector<Accepted> objs_accepted(const Bvh &bvh, const Ray &r, float t_min, float t_max) {
  std::vector<Accepted> acc;
  bvh_fold(bvh, r, t_min, t_max, [&](int32_t i) {
    Hit h;
    if (sphere_hit(bvh.L[i], r, t_min, t_max, &h)) acc.push_back({h.t, i, h});
  });
  return acc;
}

// Runs fn(first, end) over spans of 64 rays on `threads` threads (<= 0: all cores).
void for_spans(int64_t n, int32_t threads, const std::function<void(int64_t, int64_t)> &fn) {
  const int64_t span = 64, nunits = (n + span - 1) / span;
  int nthreads = threads > 0 ? threads : (int)std::thread::hardware_concurrency();
  if (nthreads < 1) nthreads = 1;
  if (nthreads > nunits) nthreads = (int)std::max<int64_t>(nunits, 1);
  std::atomic<int64_t> next_unit{0};
  auto worker = [&]() {
    for (;;) {
      const int64_t unit = next_unit.fetch_add(1);
      if (unit >= nunits) break;
      fn(unit * span, std::min(n, (unit + 1) * span));
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < nthreads; t++) pool.emplace_back(worker);
  worker();
  for (auto &t : pool) t.join();
}

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

// objs_hit objs r t_min t_max per ray of rays (n x 6: origin.xyz, dir.xyz).  out8 per ray = struct ray_b200_hit: t,
// bits(sphere), p.xyz, normal.xyz, where sphere = perm[acc_j] is the index into the scene's sphere array; no hit:
// t = -1, sphere = -1, p = normal = 0.
int oracle_trace_hits(void *pv, const float *rays, int64_t n, float t_min, float t_max, float *out8, int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays + 6 * i;
      const Ray r = {{q[0], q[1], q[2]}, {q[3], q[4], q[5]}};
      Hit h;
      int32_t leaf = -1;
      float *o = out8 + 8 * i;
      if (objs_hit_leaf(p->objs, r, t_min, t_max, &h, &leaf)) {
        const int32_t sphere = p->objs.perm[(size_t)leaf];
        o[0] = h.t; memcpy(o + 1, &sphere, 4);
        o[2] = h.p.x; o[3] = h.p.y; o[4] = h.p.z; o[5] = h.normal.x; o[6] = h.normal.y; o[7] = h.normal.z;
      } else {
        const int32_t none = -1;
        o[0] = -1.0f; memcpy(o + 1, &none, 4);
        for (int k = 2; k < 8; k++) o[k] = 0.0f;
      }
    }
  });
  return 0;
}

// ray_colour objs r max_depth (ray.fut:126-148) per ray: out_rgb n x 3; out_segments (optional) = its objs_hit calls.
int oracle_trace_paths(void *pv, const float *rays, int64_t n, int32_t max_depth, float *out_rgb, int32_t *out_segments,
                       int32_t threads) {
  Prepared *p = (Prepared *)pv;
  if (!p || n < 0) return 1;
  for_spans(n, threads, [&](int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; i++) {
      const float *q = rays + 6 * i;
      Counters cn;
      const V3 c = ray_colour(p->objs, Ray{{q[0], q[1], q[2]}, {q[3], q[4], q[5]}}, max_depth, &cn);
      out_rgb[3 * i] = c.x; out_rgb[3 * i + 1] = c.y; out_rgb[3 * i + 2] = c.z;
      if (out_segments) out_segments[i] = (int32_t)cn.segments;
    }
  });
  return 0;
}

// get_ray (ray.fut:109-114) of the prepared camera for sample s of pixel (row j, column i), as oracle_render makes it:
// out6 = origin, dir
void oracle_camera_ray(void *pv, int64_t h, int64_t w, int32_t spp, int64_t j, int64_t i, int32_t s, float *out6) {
  Prepared *p = (Prepared *)pv;
  float ox, oy;
  sample_offset(s, &ox, &oy);
  float u = ((float)i + ox) / (float)w;
  float v = ((float)(h - j) + oy) / (float)h;
  if (spp == 1) { u = (float)i / (float)w; v = (float)(h - j) / (float)h; }
  const Ray r = get_ray(p->cam, u, v);
  const float o[6] = {r.origin.x, r.origin.y, r.origin.z, r.dir.x, r.dir.y, r.dir.z};
  std::copy(o, o + 6, out6);
}

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
