// C ABI, part 2: scenes and prepared scenes - the opaque types with store / restore, the entries rgbbox, irreg and
// prepare_scene (device LBVH build by default, the host builder as the independent second implementation), custom and
// random scenes, introspection (info / dump / packed), re-upload, and the host-only setup entry points.
#include "api_internal.h"

using namespace rayb200_api;

namespace {

int acquire_pinned(futhark_context *ctx, futhark_opaque_prepared_scene *p, size_t bytes) {
  if (p->pinned && p->pinned_bytes >= bytes) {
    CUDA_TRY(ctx, cudaEventSynchronize(p->pinned_event));
    return 0;
  }
  if (p->pinned) {
    CUDA_TRY(ctx, cudaEventSynchronize(p->pinned_event));
    CUDA_TRY(ctx, cudaFreeHost(p->pinned));
    p->pinned = nullptr;
  }
  for (size_t k = 0; k < ctx->pinned_cache.size(); k++) {
    auto &b = ctx->pinned_cache[k];
    if (b.bytes >= bytes && (b.bytes <= 2 * bytes + 4096 || b.bytes <= ((size_t)1 << 20))) {
      CUDA_TRY(ctx, cudaEventSynchronize(b.last_use));  // the copy that last read this block has finished
      if (p->pinned_event) cudaEventDestroy(p->pinned_event);
      p->pinned = b.ptr; p->pinned_bytes = b.bytes; p->pinned_event = b.last_use;
      ctx->pinned_cache.erase(ctx->pinned_cache.begin() + (long)k);
      return 0;
    }
  }
  CUDA_TRY(ctx, cudaMallocHost(&p->pinned, bytes + 64));
  p->pinned_bytes = bytes + 64;
  if (!p->pinned_event) CUDA_TRY(ctx, cudaEventCreateWithFlags(&p->pinned_event, cudaEventDisableTiming));
  return 0;
}

// prepare_scene, device path (default): H2D of the sphere records from page-locked memory, then the whole
// LBVH build + packing as kernels on the context's stream (bvh_build.cu).
double now_us() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e6 + ts.tv_nsec * 1e-3;
}

}  // namespace

namespace rayb200_api {

// Gives the scene's device block back to the stream-ordered pool.  Frames may still be reading it on either lane
// (pipelined submission does not join the lanes): if the scene was ever rendered on the second lane, the free goes to
// the context's reclaim stream behind the last use on both lanes; the context's stream itself is never made to wait.
int release_scene_block(futhark_context *ctx, futhark_opaque_prepared_scene *p, bool drop_order) {
  if (!p->dev.block) return 0;
  cudaStream_t where = ctx->stream;   // only ever used in the context's stream order: free there
  if (p->used[1]) {
    if (!ctx->reclaim) CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ctx->reclaim, cudaStreamNonBlocking));
    for (int l = 0; l < 2; l++)
      if (p->used[l]) CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->reclaim, p->last_use[l], 0));
    where = ctx->reclaim;
  }
  CUDA_TRY(ctx, cudaFreeAsync(p->dev.block, where));
  // The learned claim order stays: a prepared scene's spheres and camera never change (ray_b200_prepared_reupload builds
  // the same tree again), so what the recording frame measured remains true.  When the object itself goes
  // (`drop_order`), its table is freed behind the same frames as the scene.
  if (drop_order) {
    if (p->order_cache.cost) CUDA_TRY(ctx, cudaFreeAsync(p->order_cache.cost, where));
    if (p->order_cache.ready) cudaEventDestroy(p->order_cache.ready);
    p->order_cache = futhark_opaque_prepared_scene::OrderCache();
  }
  p->dev = DeviceBvh();
  if (drop_order) p->used[0] = p->used[1] = false;
  return 0;
}

void free_prepared_device(futhark_context *ctx, futhark_opaque_prepared_scene *p) {
  cudaSetDevice(ctx->cfg.device);
  release_scene_block(ctx, p, true);
  for (int l = 0; l < 2; l++)
    if (p->last_use[l]) { cudaEventDestroy(p->last_use[l]); p->last_use[l] = nullptr; }

  if (p->pinned) {
    if (ctx->pinned_cache.size() < 4) ctx->pinned_cache.push_back({p->pinned, p->pinned_bytes, p->pinned_event});
    else { cudaEventSynchronize(p->pinned_event); cudaEventDestroy(p->pinned_event); cudaFreeHost(p->pinned); }
  }
  p->dev = DeviceBvh();
  p->pinned = nullptr;
  p->pinned_event = nullptr;
}

// A page-locked staging buffer of at least `bytes`, reusing a cached one when possible (main.c frees and

int prepare_on_device(futhark_context *ctx, futhark_opaque_prepared_scene *p) {
  const bool timing = ctx->cfg.debugging != 0;
  const double t0 = timing ? now_us() : 0.0;
  const size_t n = p->host.spheres.size();
  const size_t sph_bytes = n * sizeof(SphereRec);
  if (acquire_pinned(ctx, p, sph_bytes)) return 1;
  memcpy(p->pinned, p->host.spheres.data(), sph_bytes);
  float *d_spheres = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&d_spheres, sph_bytes, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_spheres, p->pinned, sph_bytes, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaEventRecord(p->pinned_event, ctx->stream));
  const double t1 = timing ? now_us() : 0.0;
  p->refit_sweeps = (int32_t)log2f((float)(int64_t)n) + 2;  // bvh.fut:47, host libm as in the reference's C backend
  if (release_scene_block(ctx, p, false)) return 1;
  CUDA_TRY(ctx, build_bvh_device(d_spheres, (int64_t)n, p->refit_sweeps, p->dev, ctx->d_build_result, ctx->stream, &ctx->launches));
  CUDA_TRY(ctx, cudaFreeAsync(d_spheres, ctx->stream));
  // the host needs the tree depth (stack sizing) and the root box (kernel parameter) before the first render
  const double t2 = timing ? now_us() : 0.0;
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_build_result, ctx->d_build_result, sizeof(BvhBuildResult), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (timing)
    fprintf(ctx->log ? ctx->log : stderr, "[ray_b200] prepare_scene n=%zu: stage+H2D enqueue %.0f us, build enqueue %.0f us, wait %.0f us\n", n,
            t1 - t0, t2 - t1, now_us() - t2);
  memcpy(p->root_box, ctx->h_build_result->root_box, sizeof p->root_box);
  p->max_depth = ctx->h_build_result->max_depth;
  p->stale_nodes = ctx->h_build_result->stale_nodes;
  p->n = (int64_t)n;
  p->host_built = false;
  return 0;
}

// prepare_scene, host path (RAY_HOST_BUILD=1 / tuning "host_build"): scene_host.cpp builds and packs, one H2D copy.
// Kept as an independent implementation the device path is tested against.
int prepare_on_host(futhark_context *ctx, futhark_opaque_prepared_scene *p) {
  Lbvh tree;
  std::string err;
  if (!build_lbvh(p->host, tree, &err)) { set_error(ctx, "%s", err.c_str()); return 1; }
  PackedBvh pk;
  pack_bvh(p->host, tree, pk);
  const int64_t n = tree.n;
  const size_t total = device_bvh_bytes(n);
  if (acquire_pinned(ctx, p, total)) return 1;
  DeviceBvh hostside;  // the same carving, applied to the page-locked buffer
  carve_device_bvh(p->pinned, n, hostside);
  const size_t ni = (size_t)(n - 1);
  memcpy(hostside.nodes, pk.nodes.data(), ni * 64);
  memcpy(hostside.nodes_soa, pk.nodes_soa.data(), ni * 64);
  memcpy(hostside.geom, pk.geom.data(), (size_t)n * 16);
  memcpy(hostside.colour, pk.colour.data(), (size_t)n * 16);
  memcpy(hostside.morton, tree.morton.data(), (size_t)n * 4);
  memcpy(hostside.perm, tree.perm.data(), (size_t)n * 4);
  memcpy(hostside.left, tree.left.data(), ni * 4);
  memcpy(hostside.right, tree.right.data(), ni * 4);
  memcpy(hostside.parent, tree.parent.data(), ni * 4);
  memcpy(hostside.boxes, tree.boxes.data(), ni * 24);
  if (release_scene_block(ctx, p, false)) return 1;
  unsigned char *blk = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&blk, total, ctx->stream));
  carve_device_bvh(blk, n, p->dev);
  CUDA_TRY(ctx, cudaMemcpyAsync(blk, p->pinned, total, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaEventRecord(p->pinned_event, ctx->stream));
  memcpy(p->root_box, pk.root_box, sizeof p->root_box);
  p->max_depth = tree.max_depth; p->stale_nodes = tree.stale_nodes; p->refit_sweeps = tree.refit_sweeps;
  p->n = n;
  p->host_built = true;
  return 0;
}

int prepare_any(futhark_context *ctx, futhark_opaque_prepared_scene *p) {
  const int64_t n = (int64_t)p->host.spheres.size();
  if (n < 2) { set_error(ctx, "prepare_scene: a scene needs at least 2 spheres (the reference indexes I[0], bvh.fut:65)"); return 1; }
  if (n > (int64_t)1 << 26) { set_error(ctx, "prepare_scene: too many spheres (this build packs leaf indices into 26 bits)"); return 1; }
  return ctx->cfg.host_build ? prepare_on_host(ctx, p) : prepare_on_device(ctx, p);
}

}  // namespace rayb200_api

extern "C" {

// ------------------------------------------------------------------------------------------ opaque scene
int futhark_free_opaque_scene(struct futhark_context *ctx, struct futhark_opaque_scene *obj) { (void)ctx; delete obj; return 0; }

namespace {
constexpr uint32_t kSceneMagic = 0x53423252u;     // "R2BS"
constexpr uint32_t kPreparedMagic = 0x50423252u;  // "R2BP"
size_t scene_blob_size(const HostScene &s) { return 16 + 7 * sizeof(float) + s.spheres.size() * sizeof(SphereRec); }
void scene_to_blob(const HostScene &s, unsigned char *p, uint32_t magic) {
  const uint64_t n = s.spheres.size();
  memcpy(p, &magic, 4); uint32_t ver = 1; memcpy(p + 4, &ver, 4); memcpy(p + 8, &n, 8);
  float cam[7] = {s.look_from[0], s.look_from[1], s.look_from[2], s.look_at[0], s.look_at[1], s.look_at[2], s.fov};
  memcpy(p + 16, cam, sizeof cam);
  memcpy(p + 16 + sizeof cam, s.spheres.data(), n * sizeof(SphereRec));
}
bool scene_from_blob(HostScene &s, const unsigned char *p, uint32_t magic) {
  uint32_t m, ver; uint64_t n;
  memcpy(&m, p, 4); memcpy(&ver, p + 4, 4); memcpy(&n, p + 8, 8);
  if (m != magic || ver != 1) return false;
  float cam[7];
  memcpy(cam, p + 16, sizeof cam);
  memcpy(s.look_from, cam, 12); memcpy(s.look_at, cam + 3, 12); s.fov = cam[6];
  s.spheres.resize(n);
  memcpy(s.spheres.data(), p + 16 + sizeof cam, n * sizeof(SphereRec));
  return true;
}
}  // namespace

int futhark_store_opaque_scene(struct futhark_context *ctx, const struct futhark_opaque_scene *obj, void **p, size_t *n) {
  if (!ctx || !obj || !n) return 1;
  const size_t sz = scene_blob_size(obj->host);
  *n = sz;
  if (p) {
    if (!*p) *p = malloc(sz);
    if (!*p) { set_error(ctx, "store_opaque_scene: out of memory"); return 1; }
    scene_to_blob(obj->host, (unsigned char *)*p, kSceneMagic);
  }
  return 0;
}
struct futhark_opaque_scene *futhark_restore_opaque_scene(struct futhark_context *ctx, const void *p) {
  if (!ctx || !p) return nullptr;
  futhark_opaque_scene *s = new futhark_opaque_scene;
  if (!scene_from_blob(s->host, (const unsigned char *)p, kSceneMagic)) { set_error(ctx, "restore_opaque_scene: bad blob"); delete s; return nullptr; }
  return s;
}

int futhark_free_opaque_prepared_scene(struct futhark_context *ctx, struct futhark_opaque_prepared_scene *obj) {
  if (!obj) return 0;
  if (ctx && ctx->ok) {
    std::lock_guard<std::mutex> g(ctx->mu);
    for (size_t k = 0; k < obj->peer_prepared.size() && k < ctx->peers.size(); k++)
      futhark_free_opaque_prepared_scene(ctx->peers[k], obj->peer_prepared[k]);
    cudaSetDevice(ctx->cfg.device);
    free_prepared_device(ctx, obj);  // stream-ordered: a render still using it finishes first
  }
  delete obj;
  return 0;
}
// A stored prepared scene is the scene plus the (h, w) it was prepared for; restoring re-runs prepare_scene.
int futhark_store_opaque_prepared_scene(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *obj, void **p, size_t *n) {
  if (!ctx || !obj || !n) return 1;
  const size_t sz = scene_blob_size(obj->host) + 16;
  *n = sz;
  if (p) {
    if (!*p) *p = malloc(sz);
    if (!*p) { set_error(ctx, "store_opaque_prepared_scene: out of memory"); return 1; }
    scene_to_blob(obj->host, (unsigned char *)*p, kPreparedMagic);
    memcpy((unsigned char *)*p + sz - 16, &obj->h, 8);
    memcpy((unsigned char *)*p + sz - 8, &obj->w, 8);
  }
  return 0;
}
struct futhark_opaque_prepared_scene *futhark_restore_opaque_prepared_scene(struct futhark_context *ctx, const void *p) {
  if (bad_ctx(ctx) || !p) return nullptr;
  futhark_opaque_scene tmp;
  if (!scene_from_blob(tmp.host, (const unsigned char *)p, kPreparedMagic)) { set_error(ctx, "restore_opaque_prepared_scene: bad blob"); return nullptr; }
  const size_t sz = scene_blob_size(tmp.host) + 16;
  int64_t h, w;
  memcpy(&h, (const unsigned char *)p + sz - 16, 8);
  memcpy(&w, (const unsigned char *)p + sz - 8, 8);
  futhark_opaque_prepared_scene *out = nullptr;
  if (futhark_entry_prepare_scene(ctx, &out, h, w, &tmp) != 0) return nullptr;
  return out;
}

// ------------------------------------------------------------------------------------------ entry points
int futhark_entry_rgbbox(struct futhark_context *ctx, struct futhark_opaque_scene **out0) {
  if (bad_ctx(ctx) || !out0) return 1;
  futhark_opaque_scene *s = new futhark_opaque_scene;
  make_rgbbox(s->host);
  *out0 = s;
  return 0;
}
int futhark_entry_irreg(struct futhark_context *ctx, struct futhark_opaque_scene **out0) {
  if (bad_ctx(ctx) || !out0) return 1;
  futhark_opaque_scene *s = new futhark_opaque_scene;
  make_irreg(s->host);
  *out0 = s;
  return 0;
}

int futhark_entry_prepare_scene(struct futhark_context *ctx, struct futhark_opaque_prepared_scene **out0, const int64_t h,
                                const int64_t w, const struct futhark_opaque_scene *scene) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out0 || !scene) { set_error(ctx, "prepare_scene: null argument"); return 1; }
  if (h <= 0 || w <= 0) { set_error(ctx, "prepare_scene: bad image size"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  futhark_opaque_prepared_scene *p = new futhark_opaque_prepared_scene;
  p->host = scene->host;
  p->h = h; p->w = w;
  p->cam = make_camera(p->host, h, w);
  if (prepare_any(ctx, p)) { free_prepared_device(ctx, p); delete p; return 1; }
  for (futhark_context *peer : ctx->peers) {  // the scene is replicated: every device builds its own LBVH
    futhark_opaque_prepared_scene *pp = nullptr;
    if (futhark_entry_prepare_scene(peer, &pp, h, w, scene)) {
      char *pe = futhark_context_get_error(peer);
      set_error(ctx, "prepare_scene on helper device %d: %s", peer->cfg.device, pe ? pe : "?");
      free(pe);
      for (size_t k = 0; k < p->peer_prepared.size(); k++) futhark_free_opaque_prepared_scene(ctx->peers[k], p->peer_prepared[k]);
      free_prepared_device(ctx, p); delete p;
      return 1;
    }
    p->peer_prepared.push_back(pp);
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  *out0 = p;
  return 0;
}

int ray_b200_scene_from_arrays(struct futhark_context *ctx, struct futhark_opaque_scene **out0, const float *spheres, int64_t n,
                               const float *cam7) {
  if (bad_ctx(ctx)) return 1;
  if (!out0 || !spheres || !cam7 || n < 0) { set_error(ctx, "scene_from_arrays: bad argument"); return 1; }
  futhark_opaque_scene *s = new futhark_opaque_scene;
  s->host.spheres.resize((size_t)n);
  static_assert(sizeof(SphereRec) == 7 * sizeof(float), "SphereRec must be 7 packed floats");
  memcpy(s->host.spheres.data(), spheres, (size_t)n * sizeof(SphereRec));
  memcpy(s->host.look_from, cam7, 12); memcpy(s->host.look_at, cam7 + 3, 12); s->host.fov = cam7[6];
  *out0 = s;
  return 0;
}
int ray_b200_scene_random(struct futhark_context *ctx, struct futhark_opaque_scene **out0, int64_t n, uint64_t seed) {
  if (bad_ctx(ctx)) return 1;
  if (!out0 || n < 0) { set_error(ctx, "scene_random: bad argument"); return 1; }
  futhark_opaque_scene *s = new futhark_opaque_scene;
  make_random(s->host, n, seed);
  *out0 = s;
  return 0;
}
int64_t ray_b200_scene_num_spheres(struct futhark_context *ctx, const struct futhark_opaque_scene *s) { (void)ctx; return s ? (int64_t)s->host.spheres.size() : -1; }
int ray_b200_scene_get_arrays(struct futhark_context *ctx, const struct futhark_opaque_scene *s, float *spheres, float *cam7) {
  (void)ctx;
  if (!s) return 1;
  if (spheres) memcpy(spheres, s->host.spheres.data(), s->host.spheres.size() * sizeof(SphereRec));
  if (cam7) { memcpy(cam7, s->host.look_from, 12); memcpy(cam7 + 3, s->host.look_at, 12); cam7[6] = s->host.fov; }
  return 0;
}

int ray_b200_prepared_info(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, struct ray_b200_bvh_info *info) {
  if (bad_ctx(ctx) || !p || !info) return 1;
  memset(info, 0, sizeof *info);
  info->n_leaves = p->n; info->n_inner = p->n - 1;
  info->max_depth = p->max_depth; info->refit_sweeps = p->refit_sweeps; info->stale_nodes = p->stale_nodes;
  RenderParams P;
  LaunchConfig lc;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (fill_params(ctx, p, 8, 8, 1, 0, 1, nullptr, nullptr, false, P, lc) == 0) info->smem_nodes = P.smem_nodes;
  memcpy(info->root_box, p->root_box, sizeof info->root_box);
  memcpy(info->camera, &p->cam, sizeof info->camera);
  return 0;
}
int ray_b200_prepared_dump(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, uint32_t *morton, int32_t *perm,
                           int32_t *left, int32_t *right, int32_t *parent, float *boxes) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  if (!p || !p->dev.block) { set_error(ctx, "prepared_dump: invalid prepared scene"); return 1; }
  const size_t n = (size_t)p->n, ni = n - 1;
  const cudaMemcpyKind k = cudaMemcpyDeviceToHost;
  if (morton) CUDA_TRY(ctx, cudaMemcpyAsync(morton, p->dev.morton, n * 4, k, ctx->stream));
  if (perm) CUDA_TRY(ctx, cudaMemcpyAsync(perm, p->dev.perm, n * 4, k, ctx->stream));
  if (left) CUDA_TRY(ctx, cudaMemcpyAsync(left, p->dev.left, ni * 4, k, ctx->stream));
  if (right) CUDA_TRY(ctx, cudaMemcpyAsync(right, p->dev.right, ni * 4, k, ctx->stream));
  if (parent) CUDA_TRY(ctx, cudaMemcpyAsync(parent, p->dev.parent, ni * 4, k, ctx->stream));
  if (boxes) CUDA_TRY(ctx, cudaMemcpyAsync(boxes, p->dev.boxes, ni * 24, k, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}
// The packed BVH2C arrays as they sit in HBM: nodes[(n-1)*16 floats], nodes_soa[same], geom[n*4], colour[n*4]. NULLs skipped.
int ray_b200_prepared_packed(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, float *nodes, float *nodes_soa,
                             float *geom, float *colour) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  if (!p || !p->dev.block) { set_error(ctx, "prepared_packed: invalid prepared scene"); return 1; }
  const size_t n = (size_t)p->n, ni = n - 1;
  const cudaMemcpyKind k = cudaMemcpyDeviceToHost;
  if (nodes) CUDA_TRY(ctx, cudaMemcpyAsync(nodes, p->dev.nodes, ni * 64, k, ctx->stream));
  if (nodes_soa) CUDA_TRY(ctx, cudaMemcpyAsync(nodes_soa, p->dev.nodes_soa, ni * 64, k, ctx->stream));
  if (geom) CUDA_TRY(ctx, cudaMemcpyAsync(geom, p->dev.geom, n * 16, k, ctx->stream));
  if (colour) CUDA_TRY(ctx, cudaMemcpyAsync(colour, p->dev.colour, n * 16, k, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}

int ray_b200_prepared_reupload(struct futhark_context *ctx, struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!p || !p->dev.block) { set_error(ctx, "prepared_reupload: invalid prepared scene"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  return prepare_any(ctx, p);  // H2D of the sphere records again + the device LBVH build (or the host path)
}
int64_t ray_b200_prepared_device_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p) {
  (void)ctx;
  return p ? (int64_t)p->dev.block_bytes : -1;
}
// Bytes prepare_scene / prepared_reupload copy host -> device (the sphere records on the device-build path).
int64_t ray_b200_prepared_upload_bytes(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p) {
  (void)ctx;
  if (!p) return -1;
  return p->host_built ? (int64_t)p->dev.block_bytes : (int64_t)(p->host.spheres.size() * sizeof(SphereRec));
}

// ---- host-only entry points (no context, no device): the setup-path logic, testable without a GPU ----
int ray_b200_host_scene(const char *name, int64_t n, uint64_t seed, float *spheres, int64_t capacity, float *cam7, int64_t *count) {
  HostScene s;
  if (!name) return 1;
  if (!strcmp(name, "rgbbox")) make_rgbbox(s);
  else if (!strcmp(name, "irreg")) make_irreg(s);
  else if (!strcmp(name, "random")) make_random(s, n, seed);
  else return 1;
  if (count) *count = (int64_t)s.spheres.size();
  if (spheres) {
    if (capacity < (int64_t)s.spheres.size()) return 2;
    memcpy(spheres, s.spheres.data(), s.spheres.size() * sizeof(SphereRec));
  }
  if (cam7) { memcpy(cam7, s.look_from, 12); memcpy(cam7 + 3, s.look_at, 12); cam7[6] = s.fov; }
  return 0;
}
int ray_b200_host_camera(const float *cam7, int64_t h, int64_t w, float *out12) {
  if (!cam7 || !out12 || h <= 0 || w <= 0) return 1;
  HostScene s;
  memcpy(s.look_from, cam7, 12); memcpy(s.look_at, cam7 + 3, 12); s.fov = cam7[6];
  const CameraRec c = make_camera(s, h, w);
  memcpy(out12, &c, sizeof c);
  return 0;
}
int ray_b200_host_lbvh(const float *spheres, int64_t n, uint32_t *morton, int32_t *perm, int32_t *left, int32_t *right,
                       int32_t *parent, float *boxes, int32_t *info4) {
  if (!spheres || n < 0) return 1;
  HostScene s;
  s.spheres.resize((size_t)n);
  memcpy(s.spheres.data(), spheres, (size_t)n * sizeof(SphereRec));
  Lbvh t;
  std::string err;
  if (!build_lbvh(s, t, &err)) return 2;
  if (morton) memcpy(morton, t.morton.data(), t.morton.size() * 4);
  if (perm) memcpy(perm, t.perm.data(), t.perm.size() * 4);
  if (left) memcpy(left, t.left.data(), t.left.size() * 4);
  if (right) memcpy(right, t.right.data(), t.right.size() * 4);
  if (parent) memcpy(parent, t.parent.data(), t.parent.size() * 4);
  if (boxes) memcpy(boxes, t.boxes.data(), t.boxes.size() * 4);
  if (info4) { info4[0] = t.refit_sweeps; info4[1] = t.max_depth; info4[2] = t.stale_nodes; info4[3] = 0; }
  return 0;
}
void ray_b200_host_sample_offsets(int32_t spp, float *table) {
  std::vector<float> t;
  sample_offsets(spp, t);
  memcpy(table, t.data(), t.size() * sizeof(float));
}

}  // extern "C"
