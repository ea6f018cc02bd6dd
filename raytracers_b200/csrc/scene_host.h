// Host-side scene logic of the product library: scene generators, camera, LBVH construction
// (prepare_scene) and packing into the device layout the sm_90a kernels walk.
// This is product code; it shares nothing with oracle/ (tests compare the two).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace rayb200 {

struct SphereRec {  // `sphere`, ray.fut:22-24
  float px, py, pz, cr, cg, cb, radius;
};

struct HostScene {  // `scene`, ray.fut:171-174
  std::vector<SphereRec> spheres;
  float look_from[3], look_at[3], fov;
};

struct CameraRec {  // `camera`, ray.fut:88-91
  float origin[3], llc[3], horizontal[3], vertical[3];
};

struct F4 {
  float x, y, z, w;
};

// LBVH in the reference's own (Karras) node order: node 0 is the root (radixtree.fut:11-72).
struct Lbvh {
  int64_t n = 0;                      // leaves
  std::vector<uint32_t> morton;       // sorted keys (bvh.fut:41-43)
  std::vector<int32_t> perm;          // L[k] = scene.spheres[perm[k]]
  std::vector<int32_t> left, right;   // child pointers: inner i -> i, leaf i -> ~i (bvh.fut:24)
  std::vector<int32_t> parent;        // parent(root) = -1 (radixtree.fut:66-70)
  std::vector<float> boxes;           // (n-1) x {min.xyz, max.xyz} after the fixed-count Jacobi refit (bvh.fut:47-58)
  std::vector<int32_t> depth;         // depth of every inner node, root = 0
  int32_t refit_sweeps = 0, max_depth = 0, stale_nodes = 0;
};

// Device layout ("BVH2C": both child boxes stored in the parent; nodes ordered by (depth, Karras index), so the
// first K records are the top of the tree — the device builder in bvh_build.cu produces the same order).
// Inner node k = 4 x float4:
//   q0 = {Lmin.x, Lmin.y, Lmin.z, bits(left)}   q1 = {Lmax.x, Lmax.y, Lmax.z, bits(right)}
//   q2 = {Rmin.x, Rmin.y, Rmin.z, 0}            q3 = {Rmax.x, Rmax.y, Rmax.z, 0}
// A child that is a leaf has no box in the reference (bvh.fut:84 applies `op` without `contains`);
// it is stored as [-inf, +inf]^3, which passes aabb_hit for every ray, so the node step is uniform.
// Child pointers: inner -> BFS index (>= 0), leaf i -> ~i (Morton-sorted leaf index, < 0).
struct PackedBvh {
  std::vector<F4> nodes;    // 4 * (n-1), node-major (one 64-B record per node: global/L2 fetches)
  std::vector<F4> nodes_soa;  // the same records component-major: [q0 of all][q1 of all][q2][q3] — the copy that
                              // is staged into shared memory, where a 16-B stride spreads random node indices
                              // over all bank groups (the 64-B stride of `nodes` would hit only 2 of 8)
  std::vector<F4> geom;     // n x {centre.xyz, radius}, Morton-sorted order (= bvh.L)
  std::vector<F4> colour;   // n x {r, g, b, 0}
  float root_box[6];        // the root's own box (tested once per segment)
  int32_t max_depth = 0;
};

void make_rgbbox(HostScene &s);                        // ray.fut:176-221
void make_irreg(HostScene &s);                         // ray.fut:223-237
void make_random(HostScene &s, int64_t n, uint64_t seed);  // extension, SURVEY.md §8d config 5
CameraRec make_camera(const HostScene &s, int64_t h, int64_t w);  // ray.fut:93-107 as called at ray.fut:243-244

// bvh_mk (bvh.fut:30-59).  Returns false (with *err set) if n < 2 (bvh.fut:65, SURVEY S19).
bool build_lbvh(const HostScene &s, Lbvh &out, std::string *err);
void pack_bvh(const HostScene &s, const Lbvh &t, PackedBvh &out);

// sample offsets of the spp extension (ray_b200.h header comment) for samples [s_begin, s_end);
// table[2*(s - s_begin)] = ox_s, [2*(s - s_begin)+1] = oy_s
void sample_offsets(int32_t s_begin, int32_t s_end, std::vector<float> &table);

}  // namespace rayb200
