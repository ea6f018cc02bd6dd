// Internal header of the C-ABI implementation (api_context.cu, api_scene.cu, api_render.cu, api_multigpu.cu): the
// opaque objects behind include/ray.h / include/ray_b200.h and the helpers those files share.  Not installed.
#pragma once
#include "../../include/ray_b200.h"

#include <cuda_runtime.h>

#include <cmath>
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
  struct OffsetTable { int32_t s_begin, s_end; float *dev; };
  std::vector<OffsetTable> offset_tables;   // cache per sample range [s_begin, s_end) (ensure_offsets)
  int64_t launches = 0;
  ray_b200_plan last_plan{};                // plan of the last render kernel launch (ray_b200_context_last_plan)
  WavefrontBuffers wf;                     // ray queues of the wavefront kernel (grown on demand)
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
  // lane `id` for a launch: lane 0 follows the context's stream, which ray_b200_context_set_stream may have changed
  Lane &lane(int id) { if (id == 0) lanes[0].stream = stream; return lanes[id]; }
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool pipeline = false;                // ray_b200_context_set_pipeline: batches do not join lane 1 back
  uint32_t lane_seq = 0;                // pipelined submission: frames alternate lanes across calls
  cudaStream_t reclaim = nullptr;       // scene memory is freed here, ordered after its last use on either lane
  // Proximity queries of scenes with stale boxes (api_proximity.cu): complete-box records and the refit's scratch, one
  // grow-only allocation used on lane 0 only; `prox_done` is recorded behind its last use, so that a call on another
  // stream (ray_b200_context_set_stream) waits for it before overwriting it.
  unsigned char *prox_block = nullptr;
  size_t prox_bytes = 0;
  cudaEvent_t prox_done = nullptr;
  bool profiling_paused = false;
  int64_t renders = 0;
  bool ok = false;
};

struct futhark_opaque_scene {
  HostScene host;
};

struct futhark_opaque_prepared_scene {
  HostScene host;   // kept for store/restore and re-preparation; its camera is always the scene's
  // host.spheres holds the records of the current tree.  False after a build from device memory
  // (ray_b200_prepare_scene_device / ray_b200_prepared_update): host.spheres is then empty, and whatever needs the
  // records recovers them from the device arrays (recover_spheres).
  bool host_current = true;
  int64_t h = 0, w = 0;
  CameraRec cam;
  float root_box[6];
  int32_t max_depth = 0, stale_nodes = 0, refit_sweeps = 0;
  int64_t n = 0;
  // > 1: the trees of a scene batch (ray_b200_scene_batch), `scenes` trees of n spheres in all, back to back in `dev`
  // (dev.scene_off places them); max_depth is the deepest member's, root_box and cam are unused (the kernel reads each
  // member's from dev.results / dev.cams)
  int32_t scenes = 1;
  std::vector<futhark_opaque_prepared_scene *> peer_prepared;  // single-process multi-GPU: the same scene on every helper device
  DeviceBvh dev;    // everything resident in HBM (one stream-ordered allocation): packed BVH2C + the Karras-order LBVH
  unsigned char *pinned = nullptr;     // page-locked upload buffer (sphere records, or the host-built arrays)
  size_t pinned_bytes = 0;
  cudaEvent_t pinned_event = nullptr;  // completion of the last H2D copy that read `pinned`
  bool host_built = false;
  // last render that read this scene's device memory, per lane (record_scene_use): the memory is freed / replaced
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

// The inner nodes and leaves of all of p's trees: what a launch plans over and stages
inline int64_t n_inner_of(const futhark_opaque_prepared_scene *p) { return p->n - p->scenes; }
inline int64_t n_leaves_of(const futhark_opaque_prepared_scene *p) { return p->n; }
// The refit sweeps of the reference's build of n spheres, trunc(log2f(n)) + 2 (bvh.fut:47), with the host libm as in
// the reference's C backend
inline int32_t refit_sweeps_of(int64_t n) { return (int32_t)log2f((float)n) + 2; }

// B scenes of n_0 .. n_{B-1} spheres, built and rendered together (include/ray_b200.h "scene batches")
struct ray_b200_scene_batch {
  futhark_opaque_prepared_scene scene;  // every member's tree (scene.scenes = B): planned, launched and released as one scene
  int64_t h = 0, w = 0;                 // of the build: the cameras' aspect ratio
  std::vector<float> cams7;             // [B][7] the members' cameras as given
  std::vector<BvhBuildResult> results;  // [B] each member's root box, depth and stale count
  std::vector<int64_t> off;             // [B + 1] where each member's spheres start, as dev.scene_off (off[B] = scene.n)
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
// One pixel launch as its caller describes it: every entry point that renders fills one Frame, and fill_params and
// do_render read everything about the launch from it.
struct Frame {
  const futhark_opaque_prepared_scene *scene = nullptr;
  int64_t h = 0, w = 0;
  int32_t spp = 1;             // the samples of this launch (progressive kinds: added to each pixel)
  int32_t rank = 0, world = 1;
  int32_t *out_pix = nullptr;
  float *out_rgb = nullptr;
  bool tile_major = false;     // out_pix holds this rank's tiles, padded to ray_b200_shard_tiles_padded (do_render zeroes the tail)
  Query kind = Query::kPixels; // a pixel kind (render_params.h Query)
  RayQuery q{};                // the fields of q that kind reads (render_params.h RayQuery); fill_params sets view_tiles,
                               // the adaptive entry point sel / n_sel once allocated
};
// One render kernel as the host path sees it: its tuning name, what a launch of it needs from do_render, and its plan.
// kKernels[k] describes kernel k of enum ray_b200_kernel (entry RAY_B200_KERNEL_AUTO only names "auto"), and
// kKernels[kNumKernels] any other id.
struct KernelInfo {
  const char *name;        // tuning / RAY_KERNEL name
  bool claims_cursor;      // claims work from the lane's cursor, which is zeroed before the launch
  bool sample_buf;         // spreads a pixel's samples over its slots when it gets a finished-sample buffer ...
  bool needs_sample_buf;   // ... and cannot trace spp > 1 without one
  bool claim_order;        // claims tiles heavy-first or in the learned order when those are on
  bool self_signal;        // bumps the frame's done flag itself (last warp out); else a 1-thread kernel follows it
  bool warp_trace;         // records when each warp runs out of work (ray_b200_context_trace_warps)
  bool wavefront_queues;   // uses the context's one set of wavefront ray queues, so its frames run on lane 0 only
  // fills the LaunchConfig fields the kernel's launcher reads and P's staging split, for frame f
  int (*plan)(futhark_context *ctx, const Frame &f, RenderParams &P, LaunchConfig &lc);
};
constexpr int kNumKernels = RAY_B200_KERNEL_LANEWALK + 1;
extern const KernelInfo kKernels[];
// The parameter block of frame f and its launch plan (kernel, warps, K, node-queue cap, packet threshold, lane-walk
// slots, ...), which the caller hands to do_render with f; sets f.q.view_tiles of a kViews frame.
int fill_params(futhark_context *ctx, Frame &f, RenderParams &P, LaunchConfig &lc);
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
// Enqueues frame f, planned by fill_params into P and lc, on lane `lane` (0 = the context's stream).  `timed`: bracket
// the launch with the context's timing events.  `ff`: the frame's peer-frame protocol.
int do_render(futhark_context *ctx, const Frame &f, RenderParams &P, const LaunchConfig &lc, int lane = 0, bool timed = true, const FrameFlags *ff = nullptr);
// fill_params, then do_render: a frame planned and launched with nothing in between
int render_frame(futhark_context *ctx, Frame &f, int lane = 0, bool timed = true, const FrameFlags *ff = nullptr);
// The launches enqueued so far on lane `lane` read p's device memory (release_scene_block waits for them)
int record_scene_use(futhark_context *ctx, const futhark_opaque_prepared_scene *p, int lane);
// Records a launch (P and lc as launched, kind / ranged / q as given to launch_render or launch_warpqueue) as the
// context's last plan; the warp-queue kernel's fields come from wq_variant, which its launcher uses too.
void record_plan(futhark_context *ctx, const RenderParams &P, const LaunchConfig &lc, Query kind, bool ranged, const RayQuery &q);
// api_multigpu.cu: the single-process multi-GPU mode (RAY_GPUS > 1) of futhark_entry_render
int create_helper_contexts(futhark_context *ctx, const futhark_context_config *cfg, int ndev);
int render_multi_device(futhark_context *ctx, futhark_i32_2d *img, int64_t h, int64_t w, int32_t spp, const futhark_opaque_prepared_scene *p);
// api_scene.cu
void free_prepared_device(futhark_context *ctx, futhark_opaque_prepared_scene *p);
int release_scene_block(futhark_context *ctx, futhark_opaque_prepared_scene *p, bool drop_order);
int prepare_on_device(futhark_context *ctx, futhark_opaque_prepared_scene *p);
int prepare_any(futhark_context *ctx, futhark_opaque_prepared_scene *p);
// The device build of p from n records already on the device (d_spheres, read on the context's stream); returns after
// the 32-byte read-back.  The tree is built into a new block before p's old one is released, so a failed build leaves
// p as it was.  `drop_order`: the scene changes, so its learned claim order is dropped with the old block.
int build_on_device(futhark_context *ctx, futhark_opaque_prepared_scene *p, const float *d_spheres, int64_t n, bool drop_order);
// api_proximity.cu: drops the proximity queries' complete-box scratch (context free, futhark_context_clear_caches)
void free_proximity_scratch(futhark_context *ctx);

}  // namespace rayb200_api
