// C ABI, part 1: configuration, context life cycle, errors, tuning parameters, the i32_2d array type and the context-level
// extensions (stream, spp, kernel, shard, timing, warp trace).  No CPU fallback: without a usable sm_90 device
// futhark_context_new reports an error and every entry point fails.
#include "api_internal.h"

using namespace rayb200_api;

namespace rayb200_api {

void set_error(futhark_context *ctx, const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  free(ctx->error);
  ctx->error = strdup(buf);
  if (ctx->cfg.logging || ctx->cfg.debugging) fprintf(ctx->log ? ctx->log : stderr, "[ray_b200] error: %s\n", buf);
}

}  // namespace rayb200_api

namespace {

int env_int(const char *name, int dflt) {
  const char *v = getenv(name);
  if (!v || !*v) return dflt;
  return atoi(v);
}

// A kernel's name (kKernels) or its number
int parse_kernel(const char *v, int dflt) {
  if (!v || !*v) return dflt;
  for (int k = 0; k < kNumKernels; k++)
    if (!strcmp(v, kKernels[k].name)) return k;
  return atoi(v);
}

const char *kTuningNames[] = {"kernel", "spp", "blocks_per_sm", "smem_budget", "refill_min", "tail_from", "wq_warps", "wq_k", "wq_spread", "wq_packet", "wq_refill", "wq_ncap", "wq_low", "wf_sort", "learn_order", "long_path", "stage_cap", "lw_slots", "lw_warps", "lw_idle_min", "lw_passes", "permute", "heavy_first", "probe_segments", "host_build", "rank", "world", "gpus"};
constexpr int kNumTuning = sizeof(kTuningNames) / sizeof(kTuningNames[0]);

}  // namespace

extern "C" {

struct futhark_context_config *futhark_context_config_new(void) {
  futhark_context_config *cfg = new (std::nothrow) futhark_context_config;
  return cfg;
}
void futhark_context_config_free(struct futhark_context_config *cfg) { delete cfg; }
void futhark_context_config_set_debugging(struct futhark_context_config *cfg, int flag) { cfg->debugging = flag; }
void futhark_context_config_set_profiling(struct futhark_context_config *cfg, int flag) { cfg->profiling = flag; }
void futhark_context_config_set_logging(struct futhark_context_config *cfg, int flag) { cfg->logging = flag; }
void futhark_context_config_set_cache_file(struct futhark_context_config *cfg, const char *f) { cfg->cache_file = f ? f : ""; }
void futhark_context_config_set_device(struct futhark_context_config *cfg, const char *s) {
  if (!s) return;
  if (*s == '#') s++;
  cfg->device = atoi(s);
}
int futhark_get_tuning_param_count(void) { return kNumTuning; }
const char *futhark_get_tuning_param_name(int i) { return (i >= 0 && i < kNumTuning) ? kTuningNames[i] : nullptr; }
const char *futhark_get_tuning_param_class(int i) { return (i >= 0 && i < kNumTuning) ? "ray_b200" : nullptr; }
int futhark_context_config_set_tuning_param(struct futhark_context_config *cfg, const char *name, size_t v) {
  if (!strcmp(name, "kernel")) cfg->kernel = (int32_t)v;
  else if (!strcmp(name, "spp")) cfg->spp = (int32_t)v;
  else if (!strcmp(name, "blocks_per_sm")) cfg->blocks_per_sm = (int32_t)v;
  else if (!strcmp(name, "smem_budget")) cfg->smem_budget = (int32_t)v;
  else if (!strcmp(name, "refill_min")) cfg->refill_min = (int32_t)v;
  else if (!strcmp(name, "tail_from")) cfg->tail_from = (int32_t)v;
  else if (!strcmp(name, "wq_warps")) cfg->wq_warps = (int32_t)v;
  else if (!strcmp(name, "wq_k")) cfg->wq_k = (int32_t)v;
  else if (!strcmp(name, "wq_spread")) cfg->wq_spread = (int32_t)v;
  else if (!strcmp(name, "wq_refill")) cfg->wq_refill = (int32_t)v;
  else if (!strcmp(name, "wq_low")) cfg->wq_low = (int32_t)v;
  else if (!strcmp(name, "wq_packet")) cfg->wq_packet = (int32_t)v;  // (size_t)-1 = decide per scene
  else if (!strcmp(name, "wq_ncap")) cfg->wq_ncap = (int32_t)v;
  else if (!strcmp(name, "wf_sort")) cfg->wf_sort = (int32_t)v;
  else if (!strcmp(name, "learn_order")) cfg->learn_order = (int32_t)v;
  else if (!strcmp(name, "long_path")) cfg->long_path = (int32_t)v;
  else if (!strcmp(name, "stage_cap")) cfg->stage_cap = (int32_t)v;  // (size_t)-1 = decide per scene
  else if (!strcmp(name, "lw_slots")) cfg->lw_slots = (int32_t)v;
  else if (!strcmp(name, "lw_warps")) cfg->lw_warps = (int32_t)v;
  else if (!strcmp(name, "lw_idle_min")) cfg->lw_idle_min = (int32_t)v;
  else if (!strcmp(name, "lw_passes")) cfg->lw_passes = (int32_t)v;
  else if (!strcmp(name, "permute")) cfg->permute = (int32_t)v;
  else if (!strcmp(name, "heavy_first")) cfg->heavy_first = (int32_t)v;  // (size_t)-1 = decide per frame
  else if (!strcmp(name, "probe_segments")) cfg->probe_segments = (int32_t)v;
  else if (!strcmp(name, "host_build")) cfg->host_build = (int32_t)v;
  else if (!strcmp(name, "rank")) cfg->rank = (int32_t)v;
  else if (!strcmp(name, "world")) cfg->world = (int32_t)v;
  else if (!strcmp(name, "gpus")) cfg->gpus = (int32_t)v;
  else return 1;
  return 0;
}

struct futhark_context *futhark_context_new(struct futhark_context_config *cfg) {
  futhark_context *ctx = new (std::nothrow) futhark_context;
  if (!ctx) return nullptr;
  if (cfg) ctx->cfg = *cfg;
  // environment overrides: the only extension channel an unmodified futhark/main.c has
  const bool helper = cfg && cfg->gpus < 0;  // helper context of a single-process multi-GPU context: config is final
  if (!helper) ctx->cfg.device = env_int("RAY_DEVICE", ctx->cfg.device);
  ctx->cfg.spp = env_int("RAY_SPP", ctx->cfg.spp);
  ctx->cfg.kernel = parse_kernel(getenv("RAY_KERNEL"), ctx->cfg.kernel);
  if (!helper) ctx->cfg.rank = env_int("RAY_RANK", ctx->cfg.rank);
  if (!helper) ctx->cfg.world = env_int("RAY_WORLD", ctx->cfg.world);
  if (!(cfg && cfg->gpus < 0)) ctx->cfg.gpus = env_int("RAY_GPUS", ctx->cfg.gpus);
  ctx->cfg.blocks_per_sm = env_int("RAY_BLOCKS_PER_SM", ctx->cfg.blocks_per_sm);
  ctx->cfg.smem_budget = env_int("RAY_SMEM_BUDGET", ctx->cfg.smem_budget);
  ctx->cfg.refill_min = env_int("RAY_REFILL_MIN", ctx->cfg.refill_min);
  ctx->cfg.tail_from = env_int("RAY_TAIL_FROM", ctx->cfg.tail_from);
  ctx->cfg.wq_warps = env_int("RAY_WQ_WARPS", ctx->cfg.wq_warps);
  ctx->cfg.wq_k = env_int("RAY_WQ_K", ctx->cfg.wq_k);
  ctx->cfg.wq_spread = env_int("RAY_WQ_SPREAD", ctx->cfg.wq_spread);
  ctx->cfg.wq_packet = env_int("RAY_WQ_PACKET", ctx->cfg.wq_packet);
  ctx->cfg.wq_refill = env_int("RAY_WQ_REFILL", ctx->cfg.wq_refill);
  ctx->cfg.wq_low = env_int("RAY_WQ_LOW", ctx->cfg.wq_low);
  ctx->cfg.wq_ncap = env_int("RAY_WQ_NCAP", ctx->cfg.wq_ncap);
  ctx->cfg.stage_cap = env_int("RAY_STAGE_CAP", ctx->cfg.stage_cap);
  ctx->cfg.wf_sort = env_int("RAY_WF_SORT", ctx->cfg.wf_sort);
  ctx->cfg.learn_order = env_int("RAY_LEARN_ORDER", ctx->cfg.learn_order);
  ctx->cfg.long_path = env_int("RAY_LONG_PATH", ctx->cfg.long_path);
  ctx->cfg.lw_slots = env_int("RAY_LW_SLOTS", ctx->cfg.lw_slots);
  ctx->cfg.lw_warps = env_int("RAY_LW_WARPS", ctx->cfg.lw_warps);
  ctx->cfg.lw_idle_min = env_int("RAY_LW_IDLE_MIN", ctx->cfg.lw_idle_min);
  ctx->cfg.lw_passes = env_int("RAY_LW_PASSES", ctx->cfg.lw_passes);
  ctx->cfg.permute = env_int("RAY_PERMUTE", ctx->cfg.permute);
  ctx->cfg.heavy_first = env_int("RAY_HEAVY_FIRST", ctx->cfg.heavy_first);
  ctx->cfg.probe_segments = env_int("RAY_PROBE_SEGMENTS", ctx->cfg.probe_segments);
  ctx->cfg.host_build = env_int("RAY_HOST_BUILD", ctx->cfg.host_build);
  ctx->cfg.debugging = env_int("RAY_DEBUG", ctx->cfg.debugging);
  memset(&ctx->wf, 0, sizeof ctx->wf);

  auto fail = [&](const char *what, cudaError_t e) {
    set_error(ctx, "futhark_context_new: %s: %s (this library has no CPU fallback)", what, cudaGetErrorString(e));
    return ctx;
  };
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail("no CUDA device", e == cudaSuccess ? cudaErrorNoDevice : e);
  if (ctx->cfg.device < 0 || ctx->cfg.device >= ndev) return fail("device index out of range", cudaErrorInvalidDevice);
  if ((e = cudaSetDevice(ctx->cfg.device)) != cudaSuccess) return fail("cudaSetDevice", e);
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, ctx->cfg.device)) != cudaSuccess) return fail("cudaGetDeviceProperties", e);
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code runs on compute capability 9.0 only
    set_error(ctx, "futhark_context_new: device %d is sm_%d%d; this library is built for sm_90a (H100) only",
              ctx->cfg.device, prop.major, prop.minor);
    return ctx;
  }
  ctx->sm_count = prop.multiProcessorCount;
  ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  if ((e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
  ctx->stream = ctx->own_stream;
  if ((e = cudaEventCreate(&ctx->ev_start)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaEventCreate(&ctx->ev_stop)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaMalloc(&ctx->lanes[0].work_cursor, 64)) != cudaSuccess) return fail("cudaMalloc", e);
  if ((e = cudaMalloc(&ctx->counters, 5 * sizeof(unsigned long long))) != cudaSuccess) return fail("cudaMalloc", e);
  ctx->flag_timeouts = ctx->counters + 4;
  if ((e = cudaMemset(ctx->counters, 0, 5 * sizeof(unsigned long long))) != cudaSuccess) return fail("cudaMemset", e);
  if ((e = cudaMalloc(&ctx->d_build_result, sizeof(BvhBuildResult))) != cudaSuccess) return fail("cudaMalloc", e);
  if ((e = cudaMallocHost(&ctx->h_build_result, sizeof(BvhBuildResult))) != cudaSuccess) return fail("cudaMallocHost", e);
  if ((e = preload_default_kernels(ctx->max_smem_optin)) != cudaSuccess) return fail("loading the render kernels", e);
  // keep freed frames in the stream-ordered pool: futhark/main.c frees and re-allocates the image every run
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, ctx->cfg.device) == cudaSuccess) {
    unsigned long long keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  ctx->ok = true;
  {
    // One-time costs belong to context creation, not to the first timed prepare_scene (main.c:88-100 averages over its
    // runs): build a throw-away two-sphere scene so that the build kernels, CUB's sort kernels, the stream-ordered pool
    // and a page-locked staging block are loaded / allocated now (render kernels opt in to their shared memory on first launch).
    futhark_opaque_prepared_scene warm;
    warm.host.spheres = {SphereRec{0.0f, 0.0f, 0.0f, 1.0f, 1.0f, 1.0f, 1.0f}, SphereRec{3.0f, 0.0f, 0.0f, 1.0f, 1.0f, 1.0f, 1.0f}};
    if (prepare_on_device(ctx, &warm) != 0) {
      ctx->ok = false;  // the error message is already set
      return ctx;
    }
    free_prepared_device(ctx, &warm);
    // pre-grow the stream-ordered pool (it keeps what is freed: release threshold = max) and seed the page-locked cache
    void *grow = nullptr;
    if (cudaMallocAsync(&grow, (size_t)64 << 20, ctx->stream) == cudaSuccess) cudaFreeAsync(grow, ctx->stream);
    futhark_context::PinnedBlock seed{nullptr, (size_t)1 << 20, nullptr};
    if (cudaMallocHost(&seed.ptr, seed.bytes) == cudaSuccess && cudaEventCreateWithFlags(&seed.last_use, cudaEventDisableTiming) == cudaSuccess) {
      cudaEventRecord(seed.last_use, ctx->stream);
      ctx->pinned_cache.push_back(seed);
    }
    cudaStreamSynchronize(ctx->stream);
    cudaGetLastError();
    ctx->launches = 0;
  }
  // single-process multi-GPU: helper contexts on devices device+1 .. device+gpus-1 (api_multigpu.cu)
  if (ctx->cfg.gpus > 1 && !(cfg && cfg->gpus < 0)) create_helper_contexts(ctx, cfg, ndev);
  return ctx;
}

void futhark_context_free(struct futhark_context *ctx) {
  if (!ctx) return;
  for (futhark_context *peer : ctx->peers) futhark_context_free(peer);
  ctx->peers.clear();
  if (ctx->peer_tiles) { cudaSetDevice(ctx->cfg.device); cudaFree(ctx->peer_tiles); }
  if (ctx->peer_done) cudaEventDestroy(ctx->peer_done);
  if (ctx->gathered) { cudaSetDevice(ctx->cfg.device); cudaFree(ctx->gathered); }
  if (ctx->ev_gathered) cudaEventDestroy(ctx->ev_gathered);
  if (ctx->ok) {
    cudaSetDevice(ctx->cfg.device);
    cudaStreamSynchronize(ctx->stream);
  }
  for (auto &b : ctx->pinned_cache) { cudaEventDestroy(b.last_use); cudaFreeHost(b.ptr); }
  if (ctx->ok) free_wavefront(ctx);
  if (ctx->ok) free_proximity_scratch(ctx);
  for (auto &L : ctx->lanes) {
    if (L.sample_buf) cudaFree(L.sample_buf);
    if (L.tile_order_block) cudaFree(L.tile_order_block);
    if (L.work_cursor) cudaFree(L.work_cursor);
  }
  if (ctx->lanes[1].stream) { cudaStreamSynchronize(ctx->lanes[1].stream); cudaStreamDestroy(ctx->lanes[1].stream); }
  if (ctx->reclaim) { cudaStreamSynchronize(ctx->reclaim); cudaStreamDestroy(ctx->reclaim); }
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  for (auto &e : ctx->offset_tables) cudaFree(e.dev);
  if (ctx->counters) cudaFree(ctx->counters);
  if (ctx->warp_trace) cudaFree(ctx->warp_trace);
  if (ctx->d_build_result) cudaFree(ctx->d_build_result);
  if (ctx->h_build_result) cudaFreeHost(ctx->h_build_result);
  if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
  if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  free(ctx->error);
  delete ctx;
}

int futhark_context_sync(struct futhark_context *ctx) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  for (futhark_context *peer : ctx->peers) {
    if (futhark_context_sync(peer)) { char *pe = futhark_context_get_error(peer); set_error(ctx, "helper device: %s", pe ? pe : "?"); free(pe); return 1; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->lanes[1].stream) CUDA_TRY(ctx, cudaStreamSynchronize(ctx->lanes[1].stream));  // pipelined submission does not join it
  if (ctx->reclaim) CUDA_TRY(ctx, cudaStreamSynchronize(ctx->reclaim));
  return 0;
}

char *futhark_context_get_error(struct futhark_context *ctx) {
  if (!ctx) return nullptr;
  char *e = ctx->error;
  ctx->error = nullptr;
  return e;
}

char *futhark_context_report(struct futhark_context *ctx) {
  if (!ctx) return nullptr;
  std::lock_guard<std::mutex> g(ctx->mu);
  char buf[512];
  float ms = 0.0f;
  if (ctx->ok && ctx->have_timing) {
    cudaEventSynchronize(ctx->ev_stop);
    cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop);
  }
  snprintf(buf, sizeof buf,
           "ray_b200 %s\ndevice: %d (%d SMs)\nrenders: %lld\nkernel launches: %lld\nlast render: %.3f ms (device)\n",
           ray_b200_version(), ctx->cfg.device, ctx->sm_count, (long long)ctx->renders, (long long)ctx->launches, ms);
  return strdup(buf);
}
void futhark_context_set_logging_file(struct futhark_context *ctx, FILE *f) { if (ctx) ctx->log = f; }
void futhark_context_pause_profiling(struct futhark_context *ctx) { if (ctx) ctx->profiling_paused = true; }
void futhark_context_unpause_profiling(struct futhark_context *ctx) { if (ctx) ctx->profiling_paused = false; }
int futhark_context_clear_caches(struct futhark_context *ctx) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  cudaMemPool_t pool;
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // lane 1 always joins the context's stream before a call returns
  // grow-only scratch: finished-sample buffers, claim-order tables, wavefront ray queues, page-locked upload buffers
  for (auto &L : ctx->lanes) {
    if (L.sample_buf) cudaFree(L.sample_buf);
    if (L.tile_order_block) cudaFree(L.tile_order_block);
    L.sample_buf = nullptr; L.sample_buf_bytes = 0;
    L.tile_order_block = nullptr; L.tile_order_bytes = 0;
  }
  free_wavefront(ctx);
  free_proximity_scratch(ctx);
  for (auto &b : ctx->pinned_cache) { cudaEventDestroy(b.last_use); cudaFreeHost(b.ptr); }
  ctx->pinned_cache.clear();
  if (cudaDeviceGetDefaultMemPool(&pool, ctx->cfg.device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  return 0;
}

// ------------------------------------------------------------------------------------------ arrays
struct futhark_i32_2d *futhark_new_i32_2d(struct futhark_context *ctx, const int32_t *data, int64_t d0, int64_t d1) {
  if (bad_ctx(ctx) || d0 < 0 || d1 < 0) return nullptr;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  futhark_i32_2d *a = new futhark_i32_2d;
  a->shape[0] = d0; a->shape[1] = d1;
  const size_t bytes = (size_t)d0 * d1 * sizeof(int32_t);
  if (cudaMallocAsync(&a->dev, bytes ? bytes : 4, ctx->stream) != cudaSuccess) { set_error(ctx, "futhark_new_i32_2d: out of device memory"); delete a; return nullptr; }
  if (bytes && cudaMemcpyAsync(a->dev, data, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { set_error(ctx, "futhark_new_i32_2d: copy failed"); cudaFreeAsync(a->dev, ctx->stream); delete a; return nullptr; }
  cudaStreamSynchronize(ctx->stream);
  return a;
}
struct futhark_i32_2d *futhark_new_raw_i32_2d(struct futhark_context *ctx, void *device_ptr, int64_t d0, int64_t d1) {
  if (bad_ctx(ctx)) return nullptr;
  futhark_i32_2d *a = new futhark_i32_2d;
  a->dev = (int32_t *)device_ptr; a->shape[0] = d0; a->shape[1] = d1; a->owned = false;
  return a;
}
int futhark_free_i32_2d(struct futhark_context *ctx, struct futhark_i32_2d *arr) {
  if (bad_ctx(ctx)) return 1;
  if (!arr) return 0;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  if (arr->owned && arr->dev) CUDA_TRY(ctx, cudaFreeAsync(arr->dev, ctx->stream));
  delete arr;
  return 0;
}
int futhark_values_i32_2d(struct futhark_context *ctx, struct futhark_i32_2d *arr, int32_t *data) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  if (!arr || !data) { set_error(ctx, "futhark_values_i32_2d: null argument"); return 1; }
  const size_t bytes = (size_t)arr->shape[0] * arr->shape[1] * sizeof(int32_t);
  CUDA_TRY(ctx, cudaMemcpyAsync(data, arr->dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // main.c:130-133 reads `data` without syncing
  return 0;
}
void *futhark_values_raw_i32_2d(struct futhark_context *ctx, struct futhark_i32_2d *arr) { (void)ctx; return arr ? arr->dev : nullptr; }
const int64_t *futhark_shape_i32_2d(struct futhark_context *ctx, struct futhark_i32_2d *arr) { (void)ctx; return arr ? arr->shape : nullptr; }

int ray_b200_context_set_stream(struct futhark_context *ctx, void *s) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->stream = s ? (cudaStream_t)s : ctx->own_stream;
  return 0;
}
int ray_b200_context_set_spp(struct futhark_context *ctx, int32_t spp) {
  if (bad_ctx(ctx)) return 1;
  if (spp < 1) { set_error(ctx, "spp must be >= 1"); return 1; }
  ctx->cfg.spp = spp;
  return 0;
}
int ray_b200_context_set_kernel(struct futhark_context *ctx, int32_t k) {
  if (bad_ctx(ctx)) return 1;
  if (k < 0 || k >= kNumKernels) { set_error(ctx, "unknown kernel %d", k); return 1; }
  ctx->cfg.kernel = k;
  return 0;
}
int ray_b200_context_set_shard(struct futhark_context *ctx, int32_t rank, int32_t world) {
  if (bad_ctx(ctx)) return 1;
  if (world < 1 || rank < 0 || rank >= world) { set_error(ctx, "bad shard %d/%d", rank, world); return 1; }
  ctx->cfg.rank = rank; ctx->cfg.world = world;
  return 0;
}
int ray_b200_context_device(struct futhark_context *ctx) { return ctx ? ctx->cfg.device : -1; }
int ray_b200_context_last_render_ms(struct futhark_context *ctx, float *ms) {
  if (bad_ctx(ctx) || !ms) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);  // helper contexts of the single-process multi-GPU mode switch devices
  if (!ctx->have_timing) { set_error(ctx, "no render has been issued yet"); return 1; }
  CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_stop));
  CUDA_TRY(ctx, cudaEventElapsedTime(ms, ctx->ev_start, ctx->ev_stop));
  return 0;
}
int64_t ray_b200_context_launch_count(struct futhark_context *ctx) { return ctx ? ctx->launches : 0; }

int ray_b200_context_trace_warps(struct futhark_context *ctx, int32_t enable) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);
  if (enable && !ctx->warp_trace) {
    CUDA_TRY(ctx, cudaMalloc(&ctx->warp_trace, (1 + (size_t)ctx->sm_count * kWqMaxWarps) * sizeof(unsigned long long)));
  } else if (!enable && ctx->warp_trace) {
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(ctx, cudaFree(ctx->warp_trace));
    ctx->warp_trace = nullptr;
  }
  return 0;
}
int ray_b200_context_warp_trace(struct futhark_context *ctx, float *exit_us, int64_t capacity, int64_t *count) {
  if (bad_ctx(ctx) || !count) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaSetDevice(ctx->cfg.device);
  if (!ctx->warp_trace || ctx->trace_warps == 0) { set_error(ctx, "warp_trace: no traced warp-queue render yet"); return 1; }
  const int64_t n = (int64_t)ctx->sm_count * ctx->trace_warps;
  *count = n;
  if (!exit_us) return 0;
  if (capacity < n) { set_error(ctx, "warp_trace: capacity %lld < %lld", (long long)capacity, (long long)n); return 1; }
  std::vector<unsigned long long> h(1 + (size_t)n);
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_TRY(ctx, cudaMemcpy(h.data(), ctx->warp_trace, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n; i++) exit_us[i] = h[1 + i] > h[0] ? (float)((double)(h[1 + i] - h[0]) * 1e-3) : 0.0f;
  return 0;
}

const char *ray_b200_version(void) { return "ray_b200 0.2 (sm_90a)"; }

}  // extern "C"
