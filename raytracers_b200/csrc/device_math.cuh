// Strict-f32 device arithmetic of the render path.  Every function restates one reference function
// with the SAME operation order; the translation unit is compiled with -fmad=false (no FMA
// contraction), -prec-div=true, -prec-sqrt=true, -ftz=false, so each + - * / sqrt rounds exactly as
// the reference's Futhark multicore (C) backend does.  fmaxf/fminf are NaN-ignoring on both sides.
#pragma once
#include <cuda_runtime.h>

namespace rayb200 {

struct V3 {
  float x, y, z;
};

__device__ __forceinline__ V3 v3(float x, float y, float z) { return V3{x, y, z}; }
__device__ __forceinline__ V3 vadd(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }  // prim.fut:12
__device__ __forceinline__ V3 vsub(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }  // prim.fut:13
__device__ __forceinline__ V3 vmul(V3 a, V3 b) { return V3{a.x * b.x, a.y * b.y, a.z * b.z}; }  // prim.fut:14
__device__ __forceinline__ V3 vscale(float s, V3 v) { return V3{s * v.x, s * v.y, s * v.z}; }   // prim.fut:17-20
__device__ __forceinline__ float vdot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }  // prim.fut:22-24

struct Ray {  // ray.fut:11-12
  V3 o, d;
};

// Per-segment invariants of aabb_hit / sphere_hit: 1/dir per axis (ray.fut:55, hoisted: same inputs,
// same IEEE division, same bits) and a = dot dir dir (ray.fut:34).
struct RayInv {
  float ix, iy, iz, a;
};

__device__ __forceinline__ RayInv ray_invariants(const Ray &r) {
  RayInv q;
  q.ix = 1.0f / r.d.x;
  q.iy = 1.0f / r.d.y;
  q.iz = 1.0f / r.d.z;
  q.a = vdot(r.d, r.d);
  return q;
}

// aabb_hit box r t0 t1 (ray.fut:53-70, called at ray.fut:77 with the ORIGINAL t range: (0, 1e9) from
// ray_colour, or the interval of a ray query).
// The reference early-outs after each axis; tmin is non-decreasing, tmax non-increasing and neither
// can be NaN (fmaxf/fminf drop a NaN operand and the seeds t0 / t1 are finite), so the final test
// alone gives the same boolean.
__device__ __forceinline__ bool box_hit(float bminx, float bminy, float bminz, float bmaxx, float bmaxy,
                                        float bmaxz, const Ray &r, const RayInv &q, const float t0 = 0.0f,
                                        const float t1 = 1000000000.0f) {
  const float x0 = (bminx - r.o.x) * q.ix, x1 = (bmaxx - r.o.x) * q.ix;
  const float y0 = (bminy - r.o.y) * q.iy, y1 = (bmaxy - r.o.y) * q.iy;
  const float z0 = (bminz - r.o.z) * q.iz, z1 = (bmaxz - r.o.z) * q.iz;
  const bool sx = q.ix < 0.0f, sy = q.iy < 0.0f, sz = q.iz < 0.0f;
  float tmin = fmaxf(sx ? x1 : x0, t0);
  float tmax = fminf(sx ? x0 : x1, t1);
  tmin = fmaxf(sy ? y1 : y0, tmin);
  tmax = fminf(sy ? y0 : y1, tmax);
  tmin = fmaxf(sz ? z1 : z0, tmin);
  tmax = fminf(sz ? z0 : z1, tmax);
  return !(tmax <= tmin);
}

// The `t` that sphere_hit s r t_min t_max returns, or a negative value for #none (ray.fut:32-51).
// Valid t is always > t_min >= 0, so -1 is free to mean "no hit".
__device__ __forceinline__ float sphere_t(float cx, float cy, float cz, float radius, const Ray &r, float a,
                                          float t_min, float t_max) {
  const V3 oc = vsub(r.o, v3(cx, cy, cz));
  const float b = vdot(oc, r.d);
  const float c = vdot(oc, oc) - radius * radius;
  const float disc = b * b - a * c;
  if (!(disc > 0.0f)) return -1.0f;  // `discriminant <= 0` -> #none; a NaN disc fails every later compare too
  const float sq = sqrtf(disc);
  const float root1 = (-b - sq) / a;
  if (root1 < t_max && root1 > t_min) return root1;
  const float root2 = (-b + sq) / a;
  if (root2 < t_max && root2 > t_min) return root2;
  return -1.0f;
}

// colour_to_pixel (ray.fut:158-162)
__device__ __forceinline__ int pack_pixel(V3 c) {
  const int ir = (int)(255.99f * c.x);
  const int ig = (int)(255.99f * c.y);
  const int ib = (int)(255.99f * c.z);
  return (ir << 16) | (ig << 8) | ib;
}

}  // namespace rayb200
