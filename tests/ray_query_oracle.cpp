// TEST INFRASTRUCTURE, NOT PRODUCT CODE: the CPU oracle of the ray queries (include/ray_b200.h "ray queries").
//
// The literal restatement of the reference in oracle/oracle.cpp is compiled into this translation unit unchanged (it is
// included below), so every oracle_* entry of liboracle.so exists here too and operates on this library's own handles.
// On top of it: objs_hit for caller-supplied rays and intervals (ray.fut:76-86) reporting the winning leaf, ray_colour
// with any depth limit (ray.fut:126-148), and the camera rays of oracle_render.  tests/ray_query_oracle.py compiles it
// with oracle/Makefile's flags (strict f32: no FMA contraction, no -march, no fast-math).
#include "../oracle/oracle.cpp"

#include <functional>

namespace {

// ray.fut:76-86 objs_hit with bvh.fut:61-84 bvh_fold inlined literally, as oracle.cpp's objs_hit, plus acc_j: the
// winning leaf in Morton order (-1 = none).
bool objs_hit_leaf(const Bvh &bvh, const Ray &r, float t_min, float t_max, Hit *out, int32_t *leaf) {
  int32_t acc_j = -1;
  float acc_t = t_max;
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
      if (aabb_hit(node.aabb, r, t_min, t_max)) { rec = true; child = node.left; }   // ray.fut:77 (original t range)
    }
    if (!rec) { prev = inner_ptr(cur); cur = node.parent; }            // bvh.fut:79-80
    else if (child.tag == 1) { prev = inner_ptr(cur); cur = child.idx; }  // bvh.fut:83
    else {                                                             // bvh.fut:84: op acc i L[i]
      Hit h;
      if (sphere_hit(bvh.L[child.idx], r, scene_epsilon, acc_t, &h)) { acc_j = child.idx; acc_t = h.t; }  // ray.fut:78-81
      prev = child;
    }
  }
  *leaf = acc_j;
  if (acc_j >= 0) return sphere_hit(bvh.L[acc_j], r, t_min, acc_t + 1.0f, out);   // ray.fut:83-85
  return false;
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

}  // extern "C"
