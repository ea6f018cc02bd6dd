// Internal header of the C-ABI implementation (api_context.cu, api_scene.cu, api_render.cu, api_multigpu.cu): the
// opaque objects behind include/ray.h / include/ray_b200.h and the helpers those files share.  Not installed.
#pragma once
#include "../../include/ray_b200.h"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>
#include <string>
#include <vector>

#include "bvh_build.h"
#include "render_params.h"
#include "scene_host.h"

using namespace rayb200;

// ------------------------------------------------------------------------------------------ objects
struct futhark_context_config {
  int device = 0;
  int debugging = 0, profiling = 0, logging = 0;
  int32_t spp = 1;
  int32_t kernel = RAY_B200_KERNEL_AUTO;
  int32_t rank = 0, world = 1;
  int32_t gpus = 1;  // > 1: this ONE process drives that many devices (RAY_GPUS; the drop-in multi-GPU mode of main.c)
  int32_t blocks_per_sm = 4, smem_budget = 48 * 1024, refill_min = 8, tail_from = 8;
  int32_t wq_warps = 0 /* 0 = per scene: 32, or 24 for trees far larger than the caches */, wq_k = 0 /* 0 = per scene: 2 when the whole scene fits shared memory next to 24 warps' queues, else 1 */, wq_spread = 1, wq_packet = -1, wq_refill = 1, wq_ncap = 512, wq_low = 0 /* node queue: breadth-first below this many items; 0 = half the ring, -1 = plain LIFO */, permute = 1, host_build = 0;
  int32_t stage_cap = -1;    // warp-queue / lane-walk kernels: cap (bytes) on the shared memory used for staging the tree; what is not
                             // used stays L1 cache.  -1 = per scene: everything for trees the caches hold; for trees far larger, what
                             // keeps the kernel's shared memory under the 196 KB carve-out (32 KB of L1 left)
  int32_t wf_sort = 0;       // wavefront kernel, N4 experiment: re-sort the ray queue before bounces 1..wf_sort (0 = off)
  int32_t lw_slots = 0 /* 0 = as many (<= 64) as shared memory allows */, lw_warps = 0, lw_idle_min = 4, lw_passes = 4;
  int32_t learn_order = 1;   // warp-queue kernel: claim order learned from the first frame of the same prepared scene and geometry
                             // (long-path tiles first); 0 = off
  int32_t long_path = 4;     // ... a tile is "long" when one of its paths had at least this many segments (negative: four classes
                             // with thresholds 8x / 3x / 1x |long_path|)
  int32_t heavy_first = 0;   // pull long-path tiles to the front of the claim order: 0 off (default: the probe pass costs more than the tail it saves on one GPU), 1/2/4 = probe pixels per tile, -1 = on when spp > 1
  int32_t probe_segments = 8;
  std::string cache_file;
};

struct futhark_context {
  futhark_context_config cfg;
  std::mutex mu;
  char *error = nullptr;
  FILE *log = stderr;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  bool have_timing = false;
  int sm_count = 0, max_smem_optin = 0;
  unsigned long long *counters = nullptr;   // device [4]
  unsigned long long *flag_timeouts = nullptr;  // device: peer-frame flag waits that gave up (ray_b200_flag_status)
  int32_t flag_timeout_ms = 5000;               // of the waits render_batch enqueues for its jobs
  unsigned long long *warp_trace = nullptr; // device [1 + SMs * kWqMaxWarps] when tracing is on (ray_b200_context_trace_warps)
  int trace_warps = 0;                      // warps per CTA of the last traced launch
  float *offsets = nullptr;                 // device sample-offset table of the frame being set up (an entry of offset_tables)
  int32_t offsets_spp = 0;
  struct OffsetTable { int32_t spp; float *dev; };
  std::vector<OffsetTable> offset_tables;   // per-spp cache (ensure_offsets)
  int64_t launches = 0;
  WavefrontBuffers wf;                      // ray queues of the wavefront kernel (grown on demand)
  struct PinnedBlock { unsigned char *ptr; size_t bytes; cudaEvent_t last_use; };
  std::vector<PinnedBlock> pinned_cache;    // page-locked upload buffers of freed prepared scenes, reused by the next prepare_scene
  BvhBuildResult *d_build_result = nullptr, *h_build_result = nullptr;  // device scratch / page-locked host mirror
  // single-process multi-GPU (cfg.gpus > 1): one helper context per extra device; this context is rank 0 and owns them
  std::vector<futhark_context *> peers;
  bool is_peer = false;
  int32_t *peer_tiles = nullptr;        // helper context: this device's compact tile buffer (grow-only)
  size_t peer_tiles_bytes = 0;
  cudaEvent_t peer_done = nullptr;      // helper context: its shard has been rendered
  int32_t *gathered = nullptr;          // rank 0: [gpus][tiles_padded][32] staging for the de-tiling kernel (grow-only)
  size_t gathered_bytes = 0;
  cudaEvent_t ev_gathered = nullptr;    // rank 0: the peer copies of the last frame have read every helper's peer_tiles
  bool gather_pending = false;
  // Per-render scratch.  Lane 0 runs on the context's stream; lane 1 (own stream, created on first use) lets
  // ray_b200_render_batch keep two frames in flight so that one frame's tail is covered by the next frame's start.
  struct Lane {
    cudaStream_t stream = nullptr;             // lane 0: mirrors ctx->stream at each use
    int32_t *work_cursor = nullptr;            // device
    float4 *sample_buf = nullptr;              // warp-queue kernel, spp > 1: per-warp finished-sample colours
    size_t sample_buf_bytes = 0;
    unsigned char *tile_order_block = nullptr; // heavy-first claim order: keys, sorted keys, ids, order, cub temp (one allocation)
    size_t tile_order_bytes = 0;
    TileOrderBuffers tile_order_plan{};
  } lanes[2];
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool pipeline = false;                // ray_b200_context_set_pipeline: batches do not join lane 1 back
  uint32_t lane_seq = 0;                // pipelined submission: frames alternate lanes across calls
  cudaStream_t reclaim = nullptr;       // scene memory is freed here, ordered after its last use on either lane
  bool profiling_paused = false;
  int64_t renders = 0;
  bool ok = false;
};

struct futhark_opaque_scene {
  HostScene host;
};

struct futhark_opaque_prepared_scene {
  HostScene host;   // kept for store/restore and re-preparation
  int64_t h = 0, w = 0;
  CameraRec cam;
  float root_box[6];
  int32_t max_depth = 0, stale_nodes = 0, refit_sweeps = 0;
  int64_t n = 0;
  std::vector<futhark_opaque_prepared_scene *> peer_prepared;  // single-process multi-GPU: the same scene on every helper device
  DeviceBvh dev;    // everything resident in HBM (one stream-ordered allocation): packed BVH2C + the Karras-order LBVH
  unsigned char *pinned = nullptr;     // page-locked upload buffer (sphere records, or the host-built arrays)
  size_t pinned_bytes = 0;
  cudaEvent_t pinned_event = nullptr;  // completion of the last H2D copy that read `pinned`
  bool host_built = false;
  // last render that read this scene's device memory, per lane (recorded by do_render): the memory is freed / replaced
  // only after both (release_scene_block)
  mutable cudaEvent_t last_use[2] = {nullptr, nullptr};
  mutable bool used[2] = {false, false};
  // Learned claim order (api_render.cu, do_render): the first frame of a given geometry records the longest path of every
  // tile, later frames of the same prepared scene and geometry claim the long-path tiles first.  The scene and the camera
  // are fixed in a prepared scene, so a tile's paths are the same in every frame (main.c renders the same frame `runs` times).
  struct OrderCache {
    int64_t h = 0, w = 0;
    int32_t spp = 0, rank = 0, world = 0;
    int64_t tiles = 0;
    uint32_t *cost = nullptr;   // device [tiles]
    int32_t *order = nullptr;   // device [tiles]
    int state = 0;              // 0 empty, 1 order enqueued (the sort follows the recording frame on that frame's lane)
    cudaEvent_t ready = nullptr; // recorded behind the sort: frames on the other lane wait for it before they read `order`
  };
  mutable OrderCache order_cache;
};

struct futhark_i32_2d {
  int32_t *dev = nullptr;
  int64_t shape[2] = {0, 0};
  bool owned = true;
};

namespace rayb200_api {

using namespace rayb200;

void set_error(futhark_context *ctx, const char *fmt, ...);

#define CUDA_TRY(ctx, call)                                                                     \
  do {                                                                                          \
    cudaError_t e_ = (call);                                                                    \
    if (e_ != cudaSuccess) {                                                                    \
      set_error(ctx, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return 1;                                                                                 \
    }                                                                                           \
  } while (0)

inline bool bad_ctx(futhark_context *ctx) { return ctx == nullptr || !ctx->ok; }
constexpr int kAutoK2MinWarps = 20, kAutoK2Ncap = 256;   // warp-queue kernel, wq_k = 0: the plan for scenes that fit shared memory whole
constexpr size_t kSpreadBudget = (size_t)1 << 30;  // cap on the finished-sample buffer of the sample-spreading kernels

inline int64_t tiles_total(int64_t h, int64_t w) { return ((h + kTileH - 1) / kTileH) * ((w + kTileW - 1) / kTileW); }
inline int64_t tiles_of_rank(int64_t h, int64_t w, int32_t rank, int32_t world) {
  const int64_t t = tiles_total(h, w);
  return t / world + ((t % world) > rank ? 1 : 0);
}

// api_render.cu
int resolve_kernel(const futhark_context *ctx);
// The parameter block of one frame and its launch plan (kernel, warps, K, node-queue cap, packet threshold, lane-walk
// slots, ...), which the caller hands to do_render.  `accum` (progressive rendering, ray_b200_render_accumulate): the
// frame's samples [accum->s_begin, accum->s_begin + spp) on the warp-queue kernel, scaled by 1/(s_begin + spp).  `views`
// (ray_b200_render_views_into; rank 0 of 1): views->n_views frames of h x w, planned as one frame of all their tiles, on
// the warp-queue kernel; views->view_tiles is set here.
int fill_params(futhark_context *ctx, const futhark_opaque_prepared_scene *p, int64_t h, int64_t w, int32_t spp,
                int32_t rank, int32_t world, int32_t *out_pix, float *out_rgb, bool tile_major, RenderParams &P, LaunchConfig &lc,
                const RayQuery *accum = nullptr, RayQuery *views = nullptr);
void fill_scene_params(const futhark_opaque_prepared_scene *p, RenderParams &P);  // zeroes P, then its scene half
// The warp-queue kernel's plan for one launch (pixel frames and ray queries): rays in flight per warp (32 k), warps per
// CTA, node-queue cap and packet threshold in lc, how much of the scene is staged in shared memory in P.
int plan_warpqueue(futhark_context *ctx, const futhark_opaque_prepared_scene *p, bool will_spread, bool coherent, bool rays,
                   const char *what, RenderParams &P, LaunchConfig &lc);
int64_t cap_staging(const futhark_context *ctx, const futhark_opaque_prepared_scene *p, int64_t budget);
void split_staging(const futhark_opaque_prepared_scene *p, int64_t budget, int32_t &smem_nodes, int32_t &smem_spheres);
void free_wavefront(futhark_context *ctx);
// Peer-frame protocol of one frame (include/ray_b200.h): wait for *wait_flag >= wait_value before the kernel, bump
// *done_flag when this rank's pixels have landed.
struct FrameFlags {
  uint32_t *wait_flag = nullptr;
  uint32_t wait_value = 0;
  uint32_t *done_flag = nullptr;
};
int do_render(futhark_context *ctx, RenderParams &P, const LaunchConfig &lc, int lane_id = 0, bool timed = true,
              const FrameFlags *ff = nullptr, const futhark_opaque_prepared_scene *scene = nullptr,
              const RayQuery *accum = nullptr, const RayQuery *views = nullptr);
// api_multigpu.cu: the single-process multi-GPU mode (RAY_GPUS > 1) of futhark_entry_render
int create_helper_contexts(futhark_context *ctx, const futhark_context_config *cfg, int ndev);
int render_multi_device(futhark_context *ctx, futhark_i32_2d *img, int64_t h, int64_t w, int32_t spp, const futhark_opaque_prepared_scene *p);
// api_scene.cu
void free_prepared_device(futhark_context *ctx, futhark_opaque_prepared_scene *p);
int release_scene_block(futhark_context *ctx, futhark_opaque_prepared_scene *p, bool drop_order);
int prepare_on_device(futhark_context *ctx, futhark_opaque_prepared_scene *p);
int prepare_any(futhark_context *ctx, futhark_opaque_prepared_scene *p);

}  // namespace rayb200_api
