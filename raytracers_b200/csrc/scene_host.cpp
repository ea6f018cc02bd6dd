// Host-side scene generators, camera and LBVH build of the product library (see scene_host.h).
// Strict IEEE f32: built with -ffp-contract=off and no -march, so results are bit-identical to the
// reference's Futhark multicore backend (SURVEY.md §0 fact 3).
#include "scene_host.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <thread>

namespace rayb200 {

namespace {

// Tiny parallel-for over [0, n): used for the O(n log n)-ish passes of prepare_scene on big scenes.
template <class F>
void par_for(int64_t n, F &&f) {
  const int64_t grain = 1 << 14;
  unsigned hw = std::thread::hardware_concurrency();
  if (n <= grain || hw <= 1) {
    for (int64_t i = 0; i < n; i++) f(i);
    return;
  }
  const int64_t chunks = (n + grain - 1) / grain;
  const int nt = (int)std::min<int64_t>(hw, chunks);
  std::atomic<int64_t> next{0};
  auto work = [&]() {
    for (;;) {
      int64_t c = next.fetch_add(1);
      if (c >= chunks) return;
      const int64_t lo = c * grain, hi = std::min(n, lo + grain);
      for (int64_t i = lo; i < hi; i++) f(i);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < nt; t++) pool.emplace_back(work);
  work();
  for (auto &t : pool) t.join();
}

inline float dot3(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }  // prim.fut:22-24
inline void normalise3(const float *v, float *out) {                                                   // prim.fut:26-28
  const float s = 1.0f / sqrtf(dot3(v, v));
  out[0] = s * v[0]; out[1] = s * v[1]; out[2] = s * v[2];
}
inline void cross3(const float *a, const float *b, float *o) {                                         // prim.fut:30-33
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// Spread the low 10 bits of v so that two zero bits follow each (bvh.fut:8-13).
inline uint32_t spread10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}
inline uint32_t quantise10(float t) {  // bvh.fut:16-18: clamp(t*1024, 0, 1023) with NaN -> 0 through fmaxf
  return (uint32_t)fminf(fmaxf(t * 1024.0f, 0.0f), 1023.0f);
}

// The min / max of enclosing (prim.fut:38-45) with -0.0 below +0.0, as the device builder and the oracle define it:
// fminf / fmaxf leave the sign of a min or max of -0.0 and +0.0 open.
inline float min_num(float a, float b) { return a == b ? (std::signbit(a) ? a : b) : fminf(a, b); }
inline float max_num(float a, float b) { return a == b ? (std::signbit(a) ? b : a) : fmaxf(a, b); }

}  // namespace

// ---------------------------------------------------------------------------------- scenes
static void push_wall(HostScene &s, int axis_fixed, float fixed, int ax_a, int ax_b, float cr, float cg, float cb,
                      int64_t n, float k) {
  // tabulate_2d n n, flattened row-major (ray.fut:180-215)
  const float step = k / (float)n;
  const float rad = k / ((float)n * 2.0f);
  for (int64_t a = 0; a < n; a++)
    for (int64_t b = 0; b < n; b++) {
      float p[3];
      p[axis_fixed] = fixed;
      p[ax_a] = -k / 2.0f + step * (float)a;
      p[ax_b] = -k / 2.0f + step * (float)b;
      s.spheres.push_back(SphereRec{p[0], p[1], p[2], cr, cg, cb, rad});
    }
}

void make_rgbbox(HostScene &s) {
  const int64_t n = 10;
  const float k = 60.0f;
  s.spheres.clear();
  push_wall(s, 0, -k / 2.0f, 1, 2, 1.0f, 0.0f, 0.0f, n, k);  // leftwall  (y,z)  ray.fut:180-187
  push_wall(s, 2, -k / 2.0f, 0, 1, 1.0f, 1.0f, 0.0f, n, k);  // midwall   (x,y)  ray.fut:189-196
  push_wall(s, 0, k / 2.0f, 1, 2, 0.0f, 0.0f, 1.0f, n, k);   // rightwall (y,z)  ray.fut:198-205
  push_wall(s, 1, -k / 2.0f, 0, 2, 1.0f, 1.0f, 1.0f, n, k);  // bottom    (x,z)  ray.fut:208-215
  const float lf[3] = {0.0f, 30.0f, 30.0f}, la[3] = {0.0f, -1.0f, -1.0f};  // ray.fut:219-221
  std::memcpy(s.look_from, lf, sizeof lf);
  std::memcpy(s.look_at, la, sizeof la);
  s.fov = 75.0f;
}

void make_irreg(HostScene &s) {
  const int64_t n = 100;
  const float k = 600.0f;
  s.spheres.clear();
  const float step = k / (float)n, rad = k / ((float)n * 2.0f);
  for (int64_t x = 0; x < n; x++)      // ray.fut:226-233
    for (int64_t z = 0; z < n; z++)
      s.spheres.push_back(SphereRec{-k / 2.0f + step * (float)x, 0.0f, -k / 2.0f + step * (float)z, 1.0f, 1.0f, 1.0f, rad});
  const float lf[3] = {0.0f, 12.0f, 30.0f}, la[3] = {0.0f, 10.0f, -1.0f};  // ray.fut:234-237
  std::memcpy(s.look_from, lf, sizeof lf);
  std::memcpy(s.look_at, la, sizeof la);
  s.fov = 75.0f;
}

void make_random(HostScene &s, int64_t n, uint64_t seed) {
  uint64_t st = seed;
  auto draw = [&st]() -> float {  // splitmix64 -> top 24 bits -> [0,1)
    uint64_t z = (st += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    z ^= z >> 31;
    return (float)(z >> 40) * (1.0f / 16777216.0f);
  };
  s.spheres.resize((size_t)n);
  for (auto &sp : s.spheres) {
    sp.px = -500.0f + 1000.0f * draw(); sp.py = -500.0f + 1000.0f * draw(); sp.pz = -500.0f + 1000.0f * draw();
    sp.cr = 0.25f + 0.75f * draw(); sp.cg = 0.25f + 0.75f * draw(); sp.cb = 0.25f + 0.75f * draw();
    sp.radius = 0.5f + 1.5f * draw();
  }
  const float lf[3] = {0.0f, 0.0f, 1100.0f}, la[3] = {0.0f, 0.0f, 0.0f};
  std::memcpy(s.look_from, lf, sizeof lf);
  std::memcpy(s.look_at, la, sizeof la);
  s.fov = 75.0f;
}

CameraRec make_camera(const HostScene &s, int64_t h, int64_t w) {
  // ray.fut:243-244: camera look_from look_at (0,1,0) fov (f32 w / f32 h); body ray.fut:93-107
  const float aspect = (float)w / (float)h;
  const float vup[3] = {0.0f, 1.0f, 0.0f};
  const float theta = s.fov * (float)M_PI / 180.0f;
  const float half_height = tanf(theta / 2.0f);
  const float half_width = aspect * half_height;
  float diff[3] = {s.look_from[0] - s.look_at[0], s.look_from[1] - s.look_at[1], s.look_from[2] - s.look_at[2]};
  float wv[3], uv[3], vv[3], c[3];
  normalise3(diff, wv);
  cross3(vup, wv, c);
  normalise3(c, uv);
  cross3(wv, uv, vv);
  CameraRec cam;
  for (int a = 0; a < 3; a++) {
    cam.origin[a] = s.look_from[a];
    cam.llc[a] = ((s.look_from[a] - half_width * uv[a]) - half_height * vv[a]) - wv[a];
    cam.horizontal[a] = (2.0f * half_width) * uv[a];
    cam.vertical[a] = (2.0f * half_height) * vv[a];
  }
  return cam;
}

void sample_offsets(int32_t s_begin, int32_t s_end, std::vector<float> &table) {
  table.resize((size_t)(s_end - s_begin) * 2);
  for (int32_t s = s_begin; s < s_end; s++) {
    const float a = (float)s * 0.7548776662f, b = (float)s * 0.5698402909f;
    table[2 * (size_t)(s - s_begin)] = a - floorf(a);
    table[2 * (size_t)(s - s_begin) + 1] = b - floorf(b);
  }
}

// ---------------------------------------------------------------------------------- LBVH
bool build_lbvh(const HostScene &s, Lbvh &t, std::string *err) {
  const int64_t n = (int64_t)s.spheres.size();
  if (n < 2) {
    if (err) *err = "prepare_scene: a scene needs at least 2 spheres (the reference indexes I[0], bvh.fut:65)";
    return false;
  }
  if (n > (int64_t)1 << 30) {
    if (err) *err = "prepare_scene: too many spheres (i32 indices, radixtree.fut:24)";
    return false;
  }
  t.n = n;
  const SphereRec *sp = s.spheres.data();

  // centres of the sphere boxes (bvh.fut:31; ray.fut:28-30; prim.fut:47-50): min + 0.5*(max-min)
  std::vector<float> cx((size_t)n), cy((size_t)n), cz((size_t)n);
  par_for(n, [&](int64_t k) {
    const float r = sp[k].radius;
    const float lo[3] = {sp[k].px - r, sp[k].py - r, sp[k].pz - r};
    const float hi[3] = {sp[k].px + r, sp[k].py + r, sp[k].pz + r};
    cx[(size_t)k] = lo[0] + 0.5f * (hi[0] - lo[0]);
    cy[(size_t)k] = lo[1] + 0.5f * (hi[1] - lo[1]);
    cz[(size_t)k] = lo[2] + 0.5f * (hi[2] - lo[2]);
  });
  // six reductions (bvh.fut:32-37); fmaxf/fminf are associative and commutative on non-NaN input
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t k = 0; k < n; k++) {
    lo[0] = fminf(lo[0], cx[(size_t)k]); hi[0] = fmaxf(hi[0], cx[(size_t)k]);
    lo[1] = fminf(lo[1], cy[(size_t)k]); hi[1] = fmaxf(hi[1], cy[(size_t)k]);
    lo[2] = fminf(lo[2], cz[(size_t)k]); hi[2] = fmaxf(hi[2], cz[(size_t)k]);
  }
  // Morton keys (bvh.fut:38-41, 15-22).  A degenerate axis gives 0/0 = NaN -> coordinate 0.
  std::vector<uint32_t> key((size_t)n);
  const float ext[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
  par_for(n, [&](int64_t k) {
    const uint32_t qx = quantise10((cx[(size_t)k] - lo[0]) / ext[0]);
    const uint32_t qy = quantise10((cy[(size_t)k] - lo[1]) / ext[1]);
    const uint32_t qz = quantise10((cz[(size_t)k] - lo[2]) / ext[2]);
    key[(size_t)k] = spread10(qx) * 4u + spread10(qy) * 2u + spread10(qz);
  });
  // Stable sort by key (bvh.fut:43; radix_sort.fut:50-68 is LSD radix => stable).  Sorting the
  // 64-bit composite (key << 32 | index) is the same order and needs no comparator object.
  std::vector<uint64_t> comp((size_t)n);
  for (int64_t k = 0; k < n; k++) comp[(size_t)k] = ((uint64_t)key[(size_t)k] << 32) | (uint64_t)k;
  std::sort(comp.begin(), comp.end());
  t.morton.resize((size_t)n);
  t.perm.resize((size_t)n);
  for (int64_t k = 0; k < n; k++) {
    t.morton[(size_t)k] = (uint32_t)(comp[(size_t)k] >> 32);
    t.perm[(size_t)k] = (int32_t)(comp[(size_t)k] & 0xffffffffu);
  }

  // Karras radix tree (radixtree.fut:11-72).
  const int32_t ni = (int32_t)(n - 1);
  t.left.assign((size_t)ni, 0);
  t.right.assign((size_t)ni, 0);
  t.parent.assign((size_t)ni, -1);
  const uint32_t *M = t.morton.data();
  const int32_t nn = (int32_t)n;
  auto common_prefix = [M, nn](int32_t i, int32_t j) -> int32_t {  // delta, radixtree.fut:13-21
    if (j < 0 || j >= nn) return -1;
    const uint32_t a = M[i], b = M[j];
    if (a != b) return __builtin_clz(a ^ b);
    return 32 + __builtin_clz((uint32_t)i ^ (uint32_t)j);  // i != j here, so the xor is non-zero
  };
  par_for(ni, [&](int64_t ii) {
    const int32_t i = (int32_t)ii;
    const int32_t up = common_prefix(i, i + 1), down = common_prefix(i, i - 1);
    const int32_t d = (up > down) - (up < down);                       // :27
    const int32_t floor_cp = common_prefix(i, i - d);                  // :30
    int32_t span = 2;                                                  // :31-33
    while (common_prefix(i, i + span * d) > floor_cp) span *= 2;
    int32_t len = 0;                                                   // :36-40
    for (int32_t step = span / 2; step > 0; step /= 2)
      if (common_prefix(i, i + (len + step) * d) > floor_cp) len += step;
    const int32_t j = i + len * d;                                     // :41
    const int32_t node_cp = common_prefix(i, j);                       // :44
    int32_t split = 0;                                                 // :45-50
    for (int32_t q = 1; q <= len; q *= 2) {
      const int32_t step = (len + q * 2 - 1) / (q * 2);
      if (common_prefix(i, i + (split + step) * d) > node_cp) split += step;
    }
    const int32_t gamma = i + split * d + std::min(d, 0);              // :51
    t.left[(size_t)i] = (std::min(i, j) == gamma) ? ~gamma : gamma;          // :54-57
    t.right[(size_t)i] = (std::max(i, j) == gamma + 1) ? ~(gamma + 1) : gamma + 1;  // :59-62
  });
  for (int32_t i = 0; i < ni; i++) {                                   // parents by scatter, :66-70
    if (t.left[(size_t)i] >= 0) t.parent[(size_t)t.left[(size_t)i]] = i;
    if (t.right[(size_t)i] >= 0) t.parent[(size_t)t.right[(size_t)i]] = i;
  }

  // Fixed-count Jacobi refit from zero boxes (bvh.fut:44-58).  The sweep count can be smaller than
  // the tree height, leaving "stale" boxes; the reference renders with those, so we keep them.
  t.refit_sweeps = (int32_t)log2f((float)n) + 2;                       // :47
  std::vector<float> cur((size_t)ni * 6, 0.0f), nxt((size_t)ni * 6);
  auto child_box = [&](const std::vector<float> &src, int32_t p, float *b) {
    if (p < 0) {  // leaf: sphere_aabb of L[~p] (ray.fut:28-30)
      const SphereRec &q = sp[t.perm[(size_t)(~p)]];
      b[0] = q.px - q.radius; b[1] = q.py - q.radius; b[2] = q.pz - q.radius;
      b[3] = q.px + q.radius; b[4] = q.py + q.radius; b[5] = q.pz + q.radius;
    } else {
      std::memcpy(b, &src[(size_t)p * 6], 6 * sizeof(float));
    }
  };
  auto refit_node = [&](const std::vector<float> &src, int32_t k, float *dst) {
    float a[6], b[6];
    child_box(src, t.left[(size_t)k], a);
    child_box(src, t.right[(size_t)k], b);
    for (int c = 0; c < 3; c++) { dst[c] = min_num(a[c], b[c]); dst[3 + c] = max_num(a[3 + c], b[3 + c]); }  // prim.fut:38-45
  };
  for (int32_t sweep = 0; sweep < t.refit_sweeps; sweep++) {
    par_for(ni, [&](int64_t k) { refit_node(cur, (int32_t)k, &nxt[(size_t)k * 6]); });
    cur.swap(nxt);
  }
  t.boxes = cur;
  // diagnostics: nodes whose box is not the union of their children's final boxes
  std::atomic<int32_t> stale{0};
  par_for(ni, [&](int64_t k) {
    float b[6];
    refit_node(t.boxes, (int32_t)k, b);
    if (std::memcmp(b, &t.boxes[(size_t)k * 6], sizeof b) != 0) stale.fetch_add(1);
  });
  t.stale_nodes = stale.load();
  // depth (root = 0) of the deepest leaf: bounds the traversal stack
  std::vector<int32_t> depth((size_t)ni, 0);
  std::vector<int32_t> order;
  order.reserve((size_t)ni);
  order.push_back(0);
  int32_t maxd = 1;
  for (size_t head = 0; head < order.size(); head++) {
    const int32_t k = order[head];
    const int32_t dk = depth[(size_t)k];
    maxd = std::max(maxd, dk + 1);
    const int32_t ch[2] = {t.left[(size_t)k], t.right[(size_t)k]};
    for (int c = 0; c < 2; c++)
      if (ch[c] >= 0) { depth[(size_t)ch[c]] = dk + 1; order.push_back(ch[c]); }
  }
  t.max_depth = maxd;
  t.depth = depth;
  if ((int64_t)order.size() != ni) {
    if (err) *err = "prepare_scene: internal error, radix tree is not connected";
    return false;
  }
  return true;
}

void pack_bvh(const HostScene &s, const Lbvh &t, PackedBvh &out) {
  const int64_t n = t.n;
  const int32_t ni = (int32_t)(n - 1);
  // nodes ordered by (depth, Karras index): the first K packed nodes are the top of the tree (what the kernels
  // stage in shared memory); identical to the order the device builder produces with a stable sort by depth
  std::vector<int32_t> order((size_t)ni), newidx((size_t)ni, -1);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return t.depth[(size_t)a] < t.depth[(size_t)b]; });
  for (int32_t pos = 0; pos < ni; pos++) newidx[(size_t)order[(size_t)pos]] = pos;
  out.nodes.resize((size_t)ni * 4);
  const float inf = std::numeric_limits<float>::infinity();
  auto as_float = [](int32_t v) { float f; std::memcpy(&f, &v, 4); return f; };
  par_for(ni, [&](int64_t pos) {
    const int32_t k = order[(size_t)pos];
    F4 *q = &out.nodes[(size_t)pos * 4];
    const int32_t ch[2] = {t.left[(size_t)k], t.right[(size_t)k]};
    for (int c = 0; c < 2; c++) {
      float b[6];
      int32_t ptr;
      if (ch[c] < 0) {
        b[0] = b[1] = b[2] = -inf; b[3] = b[4] = b[5] = inf;
        ptr = ch[c];
      } else {
        std::memcpy(b, &t.boxes[(size_t)ch[c] * 6], sizeof b);
        ptr = newidx[(size_t)ch[c]];
      }
      q[2 * c + 0] = F4{b[0], b[1], b[2], c == 0 ? as_float(ptr) : 0.0f};
      q[2 * c + 1] = F4{b[3], b[4], b[5], 0.0f};
      if (c == 1) q[1].w = as_float(ptr);
    }
  });
  out.nodes_soa.resize((size_t)ni * 4);
  par_for(ni, [&](int64_t pos) {
    for (int c = 0; c < 4; c++) out.nodes_soa[(size_t)c * ni + (size_t)pos] = out.nodes[(size_t)pos * 4 + c];
  });
  out.geom.resize((size_t)n);
  out.colour.resize((size_t)n);
  par_for(n, [&](int64_t k) {
    const SphereRec &q = s.spheres[(size_t)t.perm[(size_t)k]];
    out.geom[(size_t)k] = F4{q.px, q.py, q.pz, q.radius};
    out.colour[(size_t)k] = F4{q.cr, q.cg, q.cb, 0.0f};
  });
  std::memcpy(out.root_box, &t.boxes[0], 6 * sizeof(float));
  out.max_depth = t.max_depth;
}

}  // namespace rayb200
