// C ABI, part 3: the render path - per-frame parameter block and launch plan (fill_params), launch of one frame on a
// lane (do_render), the entries render / render_spp and the render extensions (render_into, render_host, shards,
// batches with two frames in flight, de-tiling, peer-memory frames, work counters).
#include "api_internal.h"

using namespace rayb200_api;

namespace rayb200_api {

// Device copy of the sample-offset table of samples [s_begin, s_end) (SURVEY.md 8d: offset (0,0) at sample 0): a frame's
// is [0, spp), a progressive chunk's its own samples only, so a chunk far into a frame costs memory and host time in
// proportion to its length.  Tables are cached per range (render_batch mixes sample counts) and never freed while a
// frame may still read them.  A new table is copied from a page-locked staging buffer on the context's stream and the
// stream is synchronised before it is handed out, so the data has landed whichever lane's stream the reading kernel is
// launched on (a pageable cudaMemcpy on the legacy stream only guarantees staging, and nothing would order a non-blocking
// stream after its DMA).
static int ensure_offsets(futhark_context *ctx, int32_t s_begin, int32_t s_end) {
  for (auto &e : ctx->offset_tables)
    if (e.s_begin == s_begin && e.s_end == s_end) { ctx->offsets = e.dev; return 0; }
  std::vector<float> table;
  sample_offsets(s_begin, s_end, table);
  const size_t bytes = table.size() * sizeof(float);
  float *stage = nullptr, *dev = nullptr;
  CUDA_TRY(ctx, cudaMallocHost(&stage, bytes));
  memcpy(stage, table.data(), bytes);
  cudaError_t e = cudaMalloc(&dev, bytes);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dev, stage, bytes, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  cudaFreeHost(stage);
  if (e != cudaSuccess) { if (dev) cudaFree(dev); set_error(ctx, "sample-offset table upload failed: %s", cudaGetErrorString(e)); return 1; }
  if (ctx->offset_tables.size() >= 32) {  // evict the oldest; every lane is drained first, so no frame still reads it
    for (auto &L : ctx->lanes) if (L.stream) cudaStreamSynchronize(L.stream);
    cudaStreamSynchronize(ctx->stream);
    cudaFree(ctx->offset_tables.front().dev);
    ctx->offset_tables.erase(ctx->offset_tables.begin());
  }
  ctx->offset_tables.push_back({s_begin, s_end, dev});
  ctx->offsets = dev;
  return 0;
}

// Zeroes the kernel parameter block and fills its scene half from a prepared scene.
void fill_scene_params(const futhark_opaque_prepared_scene *p, RenderParams &P) {
  memset(&P, 0, sizeof P);
  P.nodes = p->dev.nodes; P.nodes_soa = p->dev.nodes_soa; P.geom = p->dev.geom; P.colour = p->dev.colour;
  P.n_inner = (int32_t)n_inner_of(p); P.n_leaves = (int32_t)n_leaves_of(p);
  P.max_depth = p->max_depth;
  memcpy(P.root_box, p->root_box, sizeof P.root_box);
}

// The launch plan every kernel's plan starts from: the kernel and the device's limits, every other field 0
static LaunchConfig launch_config(const futhark_context *ctx, int kernel) {
  LaunchConfig lc{};
  lc.kernel = kernel;
  lc.sm_count = ctx->sm_count;
  lc.max_dynamic_smem = ctx->max_smem_optin;
  return lc;
}

static_assert((int)Query::kPixels == RAY_B200_QUERY_PIXELS && (int)Query::kClosest == RAY_B200_QUERY_CLOSEST &&
                  (int)Query::kAnyHit == RAY_B200_QUERY_ANYHIT && (int)Query::kMultiHit == RAY_B200_QUERY_MULTIHIT &&
                  (int)Query::kAccumulate == RAY_B200_QUERY_ACCUMULATE && (int)Query::kViews == RAY_B200_QUERY_VIEWS &&
                  (int)Query::kAdaptive == RAY_B200_QUERY_ADAPTIVE && (int)Query::kAdaptiveVar == RAY_B200_QUERY_ADAPTIVE_VAR &&
                  (int)Query::kGBuffer == RAY_B200_QUERY_GBUFFER && (int)Query::kSceneBatch == RAY_B200_QUERY_SCENE_BATCH &&
                  (int)Query::kBatchClosest == RAY_B200_QUERY_SCENE_BATCH_CLOSEST &&
                  (int)Query::kBatchAnyHit == RAY_B200_QUERY_SCENE_BATCH_ANYHIT &&
                  (int)Query::kBatchMultiHit == RAY_B200_QUERY_SCENE_BATCH_MULTIHIT,
              "enum ray_b200_query names the values of Query");
static_assert(sizeof(struct ray_b200_plan) == 80, "struct ray_b200_plan is 16 int32 and 2 int64");

void record_plan(futhark_context *ctx, const RenderParams &P, const LaunchConfig &lc, Query kind, bool ranged, const RayQuery &q) {
  ray_b200_plan &r = ctx->last_plan;
  memset(&r, 0, sizeof r);
  r.kernel = lc.kernel;
  r.query = (int32_t)kind;
  r.ranged = ranged ? 1 : 0;
  r.smem_nodes = P.smem_nodes; r.smem_spheres = P.smem_spheres;
  r.n_inner = P.n_inner; r.n_leaves = P.n_leaves;
  r.stage_budget = lc.stage_budget;
  if (lc.kernel != RAY_B200_KERNEL_WARPQUEUE) return;
  const WqVariant v = wq_variant(P, kind, q, lc);
  r.k = v.k; r.warps = lc.wq_warps; r.ctas = (int32_t)v.ctas;
  r.spread = v.spread; r.packet = v.packet ? lc.wq_packet : 0;
  r.all_nodes = v.all_nodes; r.spheres = v.spheres;
  r.ncap = v.ncap; r.nlow = v.nlow;
  r.dynamic_smem = (int64_t)v.smem;
}

// A frame size every pixel launch accepts: work items are 32-bit, so at most 2^30 (padded) pixels per frame
static bool image_size_ok(int64_t h, int64_t w) {
  return h > 0 && w > 0 && h <= 65536 && w <= 65536 && ((h + 3) / 4) * ((w + 7) / 8) <= ((int64_t)1 << 25);
}

// Bytes of the finished-sample buffer of `spp` spread samples on `warps` warps per CTA (one CTA per SM); 0 when samples
// are not spread: one sample, more than 65535, spreading switched off, or a buffer over kSpreadBudget.  Planning asks for
// kWqMaxWarps, which bounds every plan (the warps it picks depend on whether samples are spread); do_render, for lc's.
static size_t spread_bytes(const futhark_context *ctx, int warps, int32_t spp) {
  if (spp <= 1 || spp > 65535 || !ctx->cfg.wq_spread) return 0;
  const size_t need = (size_t)ctx->sm_count * warps * kWqRing * (size_t)spp * sizeof(float4);
  return need <= kSpreadBudget ? need : 0;
}

// K0, K1, K2: a staging area of the smem_budget tuning; K1 / K2 run blocks_per_sm CTAs per SM, K1 refills at refill_min
static int plan_staging(futhark_context *ctx, const Frame &f, RenderParams &P, LaunchConfig &lc) {
  lc.blocks_per_sm = ctx->cfg.blocks_per_sm;
  lc.refill_min = ctx->cfg.refill_min;
  lc.stage_budget = std::min<int64_t>(ctx->cfg.smem_budget, ctx->max_smem_optin - 1024) - 128;
  split_staging(f.scene, lc.stage_budget, P.smem_nodes, P.smem_spheres);
  return 0;
}

// K3 frames: samples will be spread if the finished-sample buffer fits the budget (do_render allocates it; a failed
// allocation there falls back to pixel-bound samples, whose bigger slots are checked again at launch)
static int plan_warpqueue_frame(futhark_context *ctx, const Frame &f, RenderParams &P, LaunchConfig &lc) {
  const bool will_spread = !is_pixel_bound(f.kind) && spread_bytes(ctx, kWqMaxWarps, f.spp) != 0;
  // the rays a warp holds are coherent: samples of one pixel (spp > 1) or primary rays of a dense frame (a warp's tile
  // lies in one view: the density is that of a view, however many there are)
  const bool coherent = f.spp > 1 || f.h * f.w >= ((int64_t)1 << 22);
  return plan_warpqueue(ctx, f.scene, will_spread, coherent, false, "render", P, lc);
}

static int plan_streamqueue(futhark_context *ctx, const Frame &f, RenderParams &P, LaunchConfig &lc) {
  const futhark_opaque_prepared_scene *p = f.scene;
  const int k = 1;
  const int64_t per_warp = (int64_t)sq_warp_bytes(k, wq_node_capacity(k, p->max_depth));
  int64_t wq_w = ctx->cfg.wq_warps < 1 ? 24 : (ctx->cfg.wq_warps > kWqMaxWarps ? kWqMaxWarps : ctx->cfg.wq_warps);
  while (wq_w > 1 && wq_w * per_warp + 8192 > (int64_t)ctx->max_smem_optin) wq_w--;
  const int64_t budget = (int64_t)ctx->max_smem_optin - wq_w * per_warp - 512;
  if (budget < 256) { set_error(ctx, "render: stream-queue kernel does not fit shared memory (tree depth %d)", p->max_depth); return 1; }
  lc.wq_warps = (int32_t)wq_w;
  lc.wq_refill = std::min(std::max(ctx->cfg.wq_refill, 1), 32);
  lc.stage_budget = budget;
  split_staging(p, budget, P.smem_nodes, P.smem_spheres);
  return 0;
}

// K5: one CTA per SM, lw_warps warps (32 unless told otherwise) x lw_slots path slots each (48 unless told otherwise,
// 32..64); slots are given up first, then warps, until the queues leave room for staging the top of the tree
static int plan_lanewalk(futhark_context *ctx, const Frame &f, RenderParams &P, LaunchConfig &lc) {
  const futhark_opaque_prepared_scene *p = f.scene;
  const int scap = lw_stack_capacity(p->max_depth);
  int64_t w = ctx->cfg.lw_warps < 1 ? 32 : std::min<int64_t>(ctx->cfg.lw_warps, kWqMaxWarps);
  int64_t r = ctx->cfg.lw_slots < 1 ? 48 : (ctx->cfg.lw_slots >= 64 ? 64 : (ctx->cfg.lw_slots >= 48 ? 48 : 32));  // 32 / 48 / 64 are built
  const int64_t full_stage = 128 + n_inner_of(p) * 64 + n_leaves_of(p) * 16;
  const int64_t want_stage = std::min<int64_t>(full_stage, 16 * 1024);
  while (w * (int64_t)lw_warp_bytes((int)r, scap) + want_stage + 1024 > (int64_t)ctx->max_smem_optin) {
    if (r > 32) r -= 16;
    else if (w > 1) w--;
    else { set_error(ctx, "render: lane-walk kernel does not fit shared memory (tree depth %d)", p->max_depth); return 1; }
  }
  const int64_t budget = (int64_t)ctx->max_smem_optin - w * (int64_t)lw_warp_bytes((int)r, scap) - 512;
  lc.wq_warps = (int32_t)w;
  lc.lw_slots = (int32_t)r;
  lc.lw_idle_min = ctx->cfg.lw_idle_min;
  lc.lw_passes = ctx->cfg.lw_passes;
  lc.stage_budget = budget;
  split_staging(p, cap_staging(ctx, p, budget), P.smem_nodes, P.smem_spheres);
  return 0;
}

const KernelInfo kKernels[] = {  // name, claims_cursor, sample_buf, needs_sample_buf, claim_order, self_signal, warp_trace, wavefront_queues, plan
    {"auto",        false, false, false, false, false, false, false, nullptr},               // RAY_B200_KERNEL_AUTO
    {"mega",        false, false, false, false, false, false, false, plan_staging},          // K0 RAY_B200_KERNEL_MEGA
    {"persistent",  true,  false, false, false, false, false, false, plan_staging},          // K1 RAY_B200_KERNEL_PERSISTENT
    {"wavefront",   false, false, false, false, false, false, true,  plan_staging},          // K2 RAY_B200_KERNEL_WAVEFRONT
    {"warpqueue",   true,  true,  false, true,  true,  true,  false, plan_warpqueue_frame},  // K3 RAY_B200_KERNEL_WARPQUEUE
    {"streamqueue", true,  true,  false, false, false, false, false, plan_streamqueue},      // K4 RAY_B200_KERNEL_STREAMQUEUE
    {"lanewalk",    true,  true,  true,  false, true,  true,  false, plan_lanewalk},         // K5 RAY_B200_KERNEL_LANEWALK
    {"",            false, false, false, false, false, false, false, plan_staging},          // any other id (kernel_info)
};
static_assert(sizeof kKernels / sizeof kKernels[0] == kNumKernels + 1, "one entry per enum ray_b200_kernel, and one more");

// The tuning "kernel" and RAY_KERNEL take any number: an id outside the enum is planned with the staging plan, and
// launch_render refuses it
static const KernelInfo &kernel_info(int k) { return kKernels[k >= 0 && k < kNumKernels ? k : kNumKernels]; }

// The kernel of a pixel launch of kind `kind` and spp samples.  Every kind but kPixels runs on the warp-queue kernel, the
// fastest measured variant on every BASELINE config, and so do AUTO and a kernel that needs the finished-sample buffer
// (K5: 0.54 MB per sample on an H100) at spp > 1 when there can be none (spreading switched off, or over the budget).
static int resolve_kernel(const futhark_context *ctx, Query kind, int32_t spp) {
  const int k = kind != Query::kPixels || ctx->cfg.kernel == RAY_B200_KERNEL_AUTO ? RAY_B200_KERNEL_WARPQUEUE : ctx->cfg.kernel;
  return kernel_info(k).needs_sample_buf && spp > 1 && !spread_bytes(ctx, kWqMaxWarps, spp) ? RAY_B200_KERNEL_WARPQUEUE : k;
}

// Fills the kernel parameter block for frame f, and the frame's launch plan: that of resolve_kernel's kernel, made by its
// kKernels entry.  Every kind is planned as a frame of f.spp samples (spread or pixel-bound by that count).
// Query::kAccumulate reads the offset table of the chunk's samples [s_begin, s_end) and scales by 1/s_end.
// Query::kViews and kSceneBatch: the work items are the tiles of all q.n_views frames, so the plan (K, staging, the sample
// buffer) is that of one frame of n_views x tiles(h, w) tiles (a scene batch's over all its trees, see n_inner_of).  The adaptive kinds are planned over all tiles, an upper bound on
// their work (the selection is on the device).  A pixel-bound kind (Query::kGBuffer) is planned as a frame whose samples
// are not spread.
int fill_params(futhark_context *ctx, Frame &f, RenderParams &P, LaunchConfig &lc) {
  const futhark_opaque_prepared_scene *p = f.scene;
  const int64_t h = f.h, w = f.w; const int32_t spp = f.spp;
  const bool views = is_multi_frame(f.kind);
  if (!p || !p->dev.nodes) { set_error(ctx, "render: invalid prepared scene"); return 1; }
  if (!image_size_ok(h, w)) {
    set_error(ctx, "render: bad image size %lldx%lld", (long long)h, (long long)w);
    return 1;
  }
  if (views && tiles_total(h, w) * f.q.n_views > ((int64_t)1 << 25)) {
    // ... and per launch: at most 2^30 padded pixels over all views
    set_error(ctx, "%s: %d %s of %lldx%lld exceed 2^30 padded pixels", f.kind == Query::kViews ? "render_views" : "render_scene_batch",
              f.q.n_views, f.kind == Query::kViews ? "views" : "frames", (long long)h, (long long)w);
    return 1;
  }
  if (spp < 1) { set_error(ctx, "render: spp must be >= 1"); return 1; }
  if (f.world < 1 || f.rank < 0 || f.rank >= f.world) { set_error(ctx, "render: bad shard %d/%d", f.rank, f.world); return 1; }
  if (p->max_depth > kStackSize - 1) { set_error(ctx, "render: BVH depth %d exceeds the traversal stack", p->max_depth); return 1; }
  const int32_t s_begin = f.kind == Query::kAccumulate ? f.q.s_begin : 0, s_end = s_begin + spp;  // (the entry point keeps s_end in int32)
  const bool adaptive = is_adaptive(f.kind);
  if (!adaptive && ensure_offsets(ctx, s_begin, s_end)) return 1;
  fill_scene_params(p, P);
  // The camera depends on the aspect ratio w/h given to prepare_scene (ray.fut:243-244); render's own
  // h, w only set the pixel grid (ray.fut:246-247) — exactly as in the reference.
  memcpy(P.cam, &p->cam, sizeof P.cam);
  P.W = (int32_t)w; P.H = (int32_t)h; P.spp = spp; P.inv_spp = 1.0f / (float)s_end;
  P.offsets = adaptive ? nullptr : ctx->offsets;
  P.out_pix = f.out_pix; P.out_rgb = f.out_rgb; P.tile_major = f.tile_major ? 1 : 0;
  P.rank = f.rank; P.world = f.world;
  P.tiles_x = (int32_t)((w + kTileW - 1) / kTileW); P.tiles_y = (int32_t)((h + kTileH - 1) / kTileH);
  P.n_tiles = tiles_total(h, w);
  P.local_tiles = tiles_of_rank(h, w, f.rank, f.world);
  if (views) {  // (the entry point allows no shards)
    f.q.view_tiles = (int32_t)P.n_tiles;
    P.n_tiles = P.local_tiles = P.n_tiles * f.q.n_views;
  }
  P.n_chunks = (int32_t)((P.local_tiles + 63) / 64);
  {  // stride ~ golden ratio * n_chunks, made coprime to n_chunks
    auto gcd = [](int64_t a, int64_t b) { while (b) { const int64_t t = a % b; a = b; b = t; } return a; };
    int64_t st = std::max<int64_t>(1, (int64_t)(0.6180339887 * (double)P.n_chunks));
    while (gcd(st, P.n_chunks) != 1) st++;
    P.chunk_stride = (int32_t)(P.n_chunks > 1 ? st % P.n_chunks : 0);
    if (P.n_chunks > 1 && P.chunk_stride == 0) P.chunk_stride = 1;
    if (!ctx->cfg.permute) { P.chunk_stride = 1; }
    // modular inverse (extended Euclid): tile chunk q is claimed at position q * inv mod n_chunks (heavy-first order)
    int64_t r0 = P.n_chunks, r1 = P.chunk_stride, t0 = 0, t1 = 1;
    while (r1 != 0) {
      const int64_t qd = r0 / r1, r2 = r0 - qd * r1, t2 = t0 - qd * t1;
      r0 = r1; r1 = r2; t0 = t1; t1 = t2;
    }
    P.chunk_stride_inv = P.n_chunks > 1 ? (int32_t)(((t0 % P.n_chunks) + P.n_chunks) % P.n_chunks) : 0;
  }
  P.probes_per_tile = 1; P.probe_segments = 8;
  P.work_cursor = nullptr;  // the lane's, set by do_render
  P.counters = ctx->counters;
  P.warp_trace = nullptr;
  P.tile_order = nullptr;
  lc = launch_config(ctx, resolve_kernel(ctx, f.kind, spp));
  return kernel_info(lc.kernel).plan(ctx, f, P, lc);
}

// Shared memory not used by the warp-queue / lane-walk kernels stays L1: a tree far larger than the caches gains more from
// 60-100 KB of L1 for its hot middle levels than from a few hundred more staged top nodes.  Returns the staging budget.
int64_t cap_staging(const futhark_context *ctx, const futhark_opaque_prepared_scene *p, int64_t budget) {
  const bool huge = n_inner_of(p) * 64 > ((int64_t)8 << 20);
  // the carve-out granule below the maximum is 196 KB (sm_90: 228 KB of shared memory + L1 per SM): staying under it
  // leaves the SM 32 KB of L1 instead of ~0
  const int64_t queues = (int64_t)ctx->max_smem_optin - 512 - budget;
  // (the driver reserves 1 KB of shared memory per CTA on top of what the kernel asks for, hence the 2 KB margin)
  const int64_t under_196k = std::max<int64_t>(1024, (int64_t)196 * 1024 - 2048 - queues);
  const int64_t cap = ctx->cfg.stage_cap >= 0 ? ctx->cfg.stage_cap : (huge ? under_196k : budget);
  return std::min<int64_t>(budget, std::max<int64_t>(cap, 256));
}

// Staging area of `budget` bytes: BFS prefix of the node array, then the sphere records if they all fit.
void split_staging(const futhark_opaque_prepared_scene *p, int64_t budget, int32_t &smem_nodes, int32_t &smem_spheres) {
  const int32_t n_inner = (int32_t)n_inner_of(p), n_leaves = (int32_t)n_leaves_of(p);
  const int64_t nodes_fit = std::max<int64_t>(0, budget / 64);
  smem_nodes = (int32_t)std::min<int64_t>(n_inner, nodes_fit);
  const int64_t left = budget - (int64_t)smem_nodes * 64;
  smem_spheres = (smem_nodes == n_inner && left >= (int64_t)n_leaves * 16) ? n_leaves : 0;
}

// The warp-queue kernel's plan for a prepared scene (pixel frames and ray queries): one CTA per SM, as many warps as asked
// for (<= 32) while their queues leave >= 8 KB for staging; deep trees need bigger node stacks, so they get fewer warps.
// `coherent`: the rays a warp holds are coherent enough for the packet walk; `rays`: no packet walk at all.  The staging
// split goes to P.smem_nodes / P.smem_spheres, the rest of the plan to lc.
int plan_warpqueue(futhark_context *ctx, const futhark_opaque_prepared_scene *p, bool will_spread, bool coherent, bool rays,
                   const char *what, RenderParams &P, LaunchConfig &lc) {
  lc = launch_config(ctx, RAY_B200_KERNEL_WARPQUEUE);
  for (int pass = 0; pass < 2; pass++) {
    // Rays in flight per warp (32 K) and node-queue cap.  wq_k = 0 (default): K = 2 with a kAutoK2Ncap-entry node queue and
    // as many warps (>= kAutoK2MinWarps) as still leave the WHOLE scene (tree + spheres) staged - a round of 64 rays has
    // relatively fewer partial batches at its end than a round of 32 (spread samples keep 4 instead of 16 bytes of
    // per-slot sample state, so 28 warps fit on rgbbox) - and K = 1 with 32 warps otherwise (a scene that is only partly
    // staged loses more from the staging space the bigger slots take than it gains from fuller batches).
    int k = ctx->cfg.wq_k == 2 ? 2 : 1;
    int ncap_cfg = ctx->cfg.wq_ncap, warps_cfg = ctx->cfg.wq_warps;
    bool auto_k2 = false;
    if (ctx->cfg.wq_k == 0 && pass == 0) {
      const int64_t scene_bytes = 128 + n_inner_of(p) * 64 + n_leaves_of(p) * 16;
      const int64_t pw2 = (int64_t)wq_warp_bytes(2, wq_node_capacity(2, p->max_depth, kAutoK2Ncap), false, will_spread);
      int64_t w2 = ((int64_t)ctx->max_smem_optin - scene_bytes - 512 - 128) / pw2;   // as many warps as still leave the scene whole
      if (w2 > kWqMaxWarps) w2 = kWqMaxWarps;
      w2 &= ~(int64_t)3;             // the same number of warps on each of the SM's four schedulers
      if (w2 >= kAutoK2MinWarps) {   // 28 warps with spread samples (80-byte slots), 24 with pixel-bound ones, on rgbbox
        k = 2;
        auto_k2 = true;
        if (warps_cfg < 1) warps_cfg = (int)w2;
        if (ctx->cfg.wq_ncap == 512) ncap_cfg = kAutoK2Ncap;   // (512 = the configured default: not set by the caller)
      }
    }
    // Packet steps pay off when item-mode node fetches are expensive (part of the tree not staged in shared memory)
    // AND the rays a warp holds are coherent.  The plan is made twice: first assuming packets, to see whether the tree
    // would be fully staged anyway.
    // (the K = 2 plan is only made for scenes that are staged whole, where packets never pay: without this the first
    // attempt below would reserve the packet stacks, find the scene no longer fits next to them and switch packets ON)
    int want_packet = rays ? 0 : ((auto_k2 && ctx->cfg.wq_packet < 0) ? 0 : ctx->cfg.wq_packet);
    int64_t per_warp = 0, wq_w = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
      const bool pk = want_packet != 0;
      per_warp = (int64_t)wq_warp_bytes(k, wq_node_capacity(k, p->max_depth, ncap_cfg), pk, will_spread);
      // 32 warps hide latency best, also for the 1 M-sphere tree (64 MB of nodes) once its staging area is capped so
      // that the SM keeps 32 KB of L1 (cap_staging)
      const int auto_warps = 32;
      wq_w = warps_cfg < 1 ? auto_warps : (warps_cfg > kWqMaxWarps ? kWqMaxWarps : warps_cfg);
      while (wq_w > 1 && wq_w * per_warp + 8192 > (int64_t)ctx->max_smem_optin) wq_w--;
      if (want_packet >= 0) break;
      const int64_t b = (int64_t)ctx->max_smem_optin - wq_w * per_warp - 512 - 128;
      const bool fully_staged = b / 64 >= n_inner_of(p);
      want_packet = (!fully_staged && coherent) ? 24 : 0;
      if (want_packet != 0) break;  // the first plan (with packets) stands
    }
    int64_t budget = (int64_t)ctx->max_smem_optin - wq_w * per_warp - 512;
    if (budget < 256) { set_error(ctx, "%s: warp-queue kernel does not fit shared memory (tree depth %d)", what, p->max_depth); return 1; }
    lc.wq_packet = want_packet > 32 ? 32 : want_packet;
    lc.wq_warps = (int32_t)wq_w;
    lc.wq_k = k;
    lc.wq_ncap = ncap_cfg;
    lc.wq_refill = std::min(std::max(ctx->cfg.wq_refill, 1), 32);
    lc.wq_low = ctx->cfg.wq_low;
    lc.stage_budget = budget;
    split_staging(p, cap_staging(ctx, p, budget), P.smem_nodes, P.smem_spheres);
    // belt and braces: the K = 2 plan is only worth anything when the scene is staged whole (a scene that just misses
    // fetches its lower nodes from L2 with half the warps); if anything above left it short, plan again with K = 1
    if (!auto_k2 || (P.smem_nodes == (int32_t)n_inner_of(p) && P.smem_spheres == (int32_t)n_leaves_of(p))) break;
  }
  return 0;
}

void free_wavefront(futhark_context *ctx) {
  WavefrontBuffers &b = ctx->wf;
  for (int q = 0; q < 2; q++) {
    if (b.ray_o[q]) cudaFree(b.ray_o[q]);
    if (b.ray_d[q]) cudaFree(b.ray_d[q]);
    if (b.light[q]) cudaFree(b.light[q]);
  }
  if (b.qlen) cudaFree(b.qlen);
  if (b.accum) cudaFree(b.accum);
  if (b.sort_keys) cudaFree(b.sort_keys);   // one block: keys, sorted keys, ids, order, cub temp
  memset(&b, 0, sizeof b);
}

// Ray queues: 2 x 48 B per local pixel (+16 B accumulator), resident for the life of the context.
int ensure_wavefront(futhark_context *ctx, int64_t items) {
  WavefrontBuffers &b = ctx->wf;
  b.tail_from = ctx->cfg.tail_from;
  if (b.capacity >= items && (ctx->cfg.wf_sort > 0) == (b.order != nullptr)) { b.sort_bounces = ctx->cfg.wf_sort; return 0; }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  free_wavefront(ctx);
  b.tail_from = ctx->cfg.tail_from;
  const size_t bytes = (size_t)items * sizeof(float4);
  for (int q = 0; q < 2; q++) {
    CUDA_TRY(ctx, cudaMalloc(&b.ray_o[q], bytes));
    CUDA_TRY(ctx, cudaMalloc(&b.ray_d[q], bytes));
    CUDA_TRY(ctx, cudaMalloc(&b.light[q], bytes));
  }
  CUDA_TRY(ctx, cudaMalloc(&b.accum, bytes));
  CUDA_TRY(ctx, cudaMalloc(&b.qlen, 2 * (kMaxDepth + 2) * sizeof(int32_t)));
  b.cursor = b.qlen + (kMaxDepth + 2);
  b.capacity = items;
  b.sort_bounces = 0;
  if (ctx->cfg.wf_sort > 0 && wavefront_sort_bytes(items) > 0) {  // N4 experiment (RAY_WF_SORT = bounces to re-sort)
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t tmp = wavefront_sort_bytes(items), col = up((size_t)items * 4);
    unsigned char *blk = nullptr;
    CUDA_TRY(ctx, cudaMalloc(&blk, 4 * col + up(tmp)));
    b.sort_keys = reinterpret_cast<uint32_t *>(blk);
    b.sort_keys_out = reinterpret_cast<uint32_t *>(blk + col);
    b.sort_ids = reinterpret_cast<int32_t *>(blk + 2 * col);
    b.order = reinterpret_cast<int32_t *>(blk + 3 * col);
    b.sort_tmp = blk + 4 * col;
    b.sort_tmp_bytes = tmp;
    b.sort_bounces = ctx->cfg.wf_sort;
  }
  return 0;
}

// The lane's scratch for sorting `tiles` tile keys into a claim order (keys, sorted keys, ids, order, cub temp: one
// allocation, grown on demand), laid out in L.tile_order_plan.
static int plan_tile_order(futhark_context *ctx, futhark_context::Lane &L, int64_t tiles) {
  const size_t n = (size_t)tiles, tmp = tile_order_sort_bytes(tiles);
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t need = 4 * up(4 * n) + up(tmp);
  if (need > L.tile_order_bytes) {
    CUDA_TRY(ctx, cudaStreamSynchronize(L.stream));
    if (L.tile_order_block) CUDA_TRY(ctx, cudaFree(L.tile_order_block));
    L.tile_order_block = nullptr; L.tile_order_bytes = 0;
    CUDA_TRY(ctx, cudaMalloc(&L.tile_order_block, need));
    L.tile_order_bytes = need;
  }
  TileOrderBuffers &tb = L.tile_order_plan;
  unsigned char *q = L.tile_order_block;
  tb.keys = reinterpret_cast<uint32_t *>(q); q += up(4 * n);
  tb.keys_sorted = reinterpret_cast<uint32_t *>(q); q += up(4 * n);
  tb.ids = reinterpret_cast<int32_t *>(q); q += up(4 * n);
  tb.order = reinterpret_cast<int32_t *>(q); q += up(4 * n);
  tb.sort_tmp = q; tb.sort_tmp_bytes = tmp;
  return 0;
}

// One frame on one lane (api_internal.h).  The progressive kinds are launched without a claim-order pass (see below);
// Query::kViews, with the camera table f.q.cams in device memory, without the learned order; the adaptive kinds, with
// their selection list f.q.sel / f.q.n_sel in device memory, as two launches: the selection pass, then the render kernel.
int do_render(futhark_context *ctx, const Frame &f, RenderParams &P, const LaunchConfig &lc, int lane_id, bool timed, const FrameFlags *ff) {
  futhark_context::Lane &L = ctx->lane(lane_id);
  if (f.tile_major) {  // ranks that own one tile fewer than the padded count leave a zeroed tail (before the timing events)
    const int64_t padded = ray_b200_shard_tiles_padded(f.h, f.w, f.world);
    if (P.local_tiles < padded)
      CUDA_TRY(ctx, cudaMemsetAsync(f.out_pix + P.local_tiles * kTilePixels, 0, (size_t)(padded - P.local_tiles) * kTilePixels * 4, L.stream));
  }
  const KernelInfo &K = kernel_info(lc.kernel);
  if (K.wavefront_queues && ensure_wavefront(ctx, P.local_tiles * kTilePixels)) return 1;
  P.sample_buf = nullptr;
  const size_t need = K.sample_buf && !is_pixel_bound(f.kind) ? spread_bytes(ctx, lc.wq_warps, P.spp) : 0;
  if (need) {
    // samples of a pixel are spread over a warp's slots; finished colours wait here for the in-order sum
    // (0.54 MB per sample on an H100's 132 SMs with 32 warps).  Above a memory budget, or when the allocation fails, the frame falls
    // back to the pixel-bound variant of the same kernel (kSpread = false), which handles any sample count.
    bool have = need <= L.sample_buf_bytes;
    if (!have) {
      CUDA_TRY(ctx, cudaStreamSynchronize(L.stream));
      if (L.sample_buf) CUDA_TRY(ctx, cudaFree(L.sample_buf));
      L.sample_buf = nullptr; L.sample_buf_bytes = 0;
      if (cudaMalloc(&L.sample_buf, need) == cudaSuccess) { L.sample_buf_bytes = need; have = true; }
      else { L.sample_buf = nullptr; cudaGetLastError(); }
    }
    P.sample_buf = have ? L.sample_buf : nullptr;
    if (!have && K.needs_sample_buf) { set_error(ctx, "render: out of device memory for the finished-sample buffer (%zu bytes)", need); return 1; }
  }
  // heavy-first claim order (K.claim_order): worth its probe pass when a frame is long enough to have a tail to lose
  // — more than one sample per pixel — and pointless when every tile is claimed in the first wave anyway.
  // A progressive or G-buffer launch uses neither this nor the learned order below (DESIGN.md, progressive rendering).  A views launch
  // probes its tiles with their views' cameras; it does not use the learned order either, which is recorded for one camera.
  const int hf = ctx->cfg.heavy_first;
  const bool heavy_first = !is_plain_order(f.kind) && K.claim_order && P.local_tiles > 1 && P.local_tiles < (1ll << 26) &&
                           (hf > 0 || (hf < 0 && P.spp > 1));
  if (heavy_first) {
    P.probes_per_tile = hf >= 4 ? 4 : (hf >= 2 ? 2 : 1);
    P.probe_segments = std::min(std::max(ctx->cfg.probe_segments, 1), kMaxDepth);
    if (plan_tile_order(ctx, L, P.local_tiles)) return 1;
    P.tile_order = L.tile_order_plan.order;
  }
  // Learned claim order (every frame of a prepared scene, single calls - the protocol of main.c, which renders the same
  // frame `runs` times - and batch frames on either lane alike).  First frame of a geometry: record the longest path per
  // tile; afterwards: long-path tiles first.  The table belongs to the prepared scene; `ready` orders its sort before
  // readers on the other lane, the scene's last-use events keep a re-recording away from frames still reading it.
  bool record_order = false;
  // (Frames of more than 2^24 tile-samples do not end on their longest paths any more, and un-mixing cheap and expensive
  // tiles costs them more than the shorter tail saves.)
  if (!heavy_first && f.kind == Query::kPixels && ctx->cfg.learn_order && K.claim_order && P.local_tiles > 64 &&
      P.local_tiles < (1ll << 26) && (ctx->cfg.learn_order > 1 || P.local_tiles * (int64_t)P.spp <= ((int64_t)1 << 24))) {
    auto &oc = f.scene->order_cache;
    const bool same = oc.state == 1 && oc.h == P.H && oc.w == P.W && oc.spp == P.spp && oc.rank == P.rank && oc.world == P.world && oc.tiles == P.local_tiles;
    if (same) {
      CUDA_TRY(ctx, cudaStreamWaitEvent(L.stream, oc.ready, 0));   // the sort may have run on the other lane
      P.tile_order = oc.order;
    } else if (oc.state == 1 && ctx->lanes[1].stream &&
               ((f.scene->used[0] && cudaEventQuery(f.scene->last_use[0]) != cudaSuccess) || (f.scene->used[1] && cudaEventQuery(f.scene->last_use[1]) != cudaSuccess))) {
      // another geometry, and frames in flight on some lane may still be reading the table of the previous one: this frame
      // renders in the plain permuted order (the table is re-recorded by the first frame that finds the scene idle)
      cudaGetLastError();
    } else {
      if (oc.tiles != P.local_tiles) {
        if (oc.cost) CUDA_TRY(ctx, cudaFreeAsync(oc.cost, L.stream));   // behind the frames that read the old table
        oc.cost = nullptr; oc.order = nullptr; oc.tiles = 0;
        CUDA_TRY(ctx, cudaMallocAsync(&oc.cost, 2 * (size_t)P.local_tiles * sizeof(uint32_t), L.stream));
        oc.order = reinterpret_cast<int32_t *>(oc.cost + P.local_tiles);
        oc.tiles = P.local_tiles;
      }
      oc.h = P.H; oc.w = P.W; oc.spp = P.spp; oc.rank = P.rank; oc.world = P.world; oc.state = 0;
      CUDA_TRY(ctx, cudaMemsetAsync(oc.cost, 0, (size_t)P.local_tiles * sizeof(uint32_t), L.stream));
      P.tile_cost = oc.cost;
      record_order = true;
      // scratch of the sort that follows the frame; the sorted order goes to the scene's table
      if (plan_tile_order(ctx, L, P.local_tiles)) return 1;
      L.tile_order_plan.order = oc.order;
    }
  }
  P.work_cursor = L.work_cursor;
  if (ctx->warp_trace && K.warp_trace && lane_id == 0) {
    const size_t n = 1 + (size_t)lc.sm_count * kWqMaxWarps;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->warp_trace, 0, n * sizeof(unsigned long long), L.stream));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->warp_trace, 0xff, sizeof(unsigned long long), L.stream));
    P.warp_trace = ctx->warp_trace;
    ctx->trace_warps = lc.wq_warps;
  }
  if (timed) CUDA_TRY(ctx, cudaEventRecord(ctx->ev_start, L.stream));
  if (K.claims_cursor) CUDA_TRY(ctx, cudaMemsetAsync(L.work_cursor, 0, 2 * sizeof(int32_t), L.stream));  // [0] work cursor, [1] departed warps
  P.frame_flag = (ff && K.self_signal) ? ff->done_flag : nullptr;
  if (ff && ff->wait_flag) launch_flag_wait(ff->wait_flag, ff->wait_value, (long long)ctx->flag_timeout_ms * 1000000ll, ctx->flag_timeouts, L.stream);
  if (heavy_first) launch_tile_order(P, L.tile_order_plan, L.stream, &ctx->launches, f.kind, f.q);
  if (is_adaptive(f.kind)) {
    CUDA_TRY(ctx, cudaMemsetAsync(f.q.n_sel, 0, sizeof(int32_t), L.stream));
    launch_adaptive_select(P, f.q, L.stream, &ctx->launches);
  }
  {
    const cudaError_t le = launch_render(P, lc, &ctx->wf, L.stream, &ctx->launches, f.kind, f.q);
    if (le == cudaErrorNotSupported) {
      set_error(ctx, "render: kernel %d is not part of this build (libray_b200.so carries mega / warpqueue; the alternatives "
                     "persistent / wavefront / streamqueue / lanewalk are in libray_b200_all.so, built with RAYB200_ALL_KERNELS)", lc.kernel);
      return 1;
    }
    CUDA_TRY(ctx, le);
    record_plan(ctx, P, lc, f.kind, false, f.q);
  }
  if (record_order) {  // after the recording frame (outside its timing events' kernel, inside the stream order): cost -> order
    launch_tile_order_from_cost(P, f.scene->order_cache.cost, ctx->cfg.long_path == 0 ? 4 : ctx->cfg.long_path, L.tile_order_plan, L.stream, &ctx->launches);
    if (!f.scene->order_cache.ready) CUDA_TRY(ctx, cudaEventCreateWithFlags(&f.scene->order_cache.ready, cudaEventDisableTiming));
    CUDA_TRY(ctx, cudaEventRecord(f.scene->order_cache.ready, L.stream));
    f.scene->order_cache.state = 1;
  }
  if (ff && ff->done_flag && !K.self_signal) launch_flag_bump(ff->done_flag, L.stream);
  CUDA_TRY(ctx, cudaGetLastError());
  if (record_scene_use(ctx, f.scene, lane_id)) return 1;
  if (timed) {
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_stop, L.stream));
    ctx->have_timing = true;
  }
  ctx->renders++;
  return 0;
}

int render_frame(futhark_context *ctx, Frame &f, int lane, bool timed, const FrameFlags *ff) {
  RenderParams P;
  LaunchConfig lc;
  return fill_params(ctx, f, P, lc) || do_render(ctx, f, P, lc, lane, timed, ff);
}

int record_scene_use(futhark_context *ctx, const futhark_opaque_prepared_scene *p, int lane) {
  if (!p->last_use[lane]) CUDA_TRY(ctx, cudaEventCreateWithFlags(&p->last_use[lane], cudaEventDisableTiming));
  CUDA_TRY(ctx, cudaEventRecord(p->last_use[lane], ctx->lanes[lane].stream));
  p->used[lane] = true;
  return 0;
}

}  // namespace rayb200_api

extern "C" {

int ray_b200_entry_render_spp(struct futhark_context *ctx, struct futhark_i32_2d **out0, int64_t h, int64_t w, int32_t spp,
                              const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out0) { set_error(ctx, "render: null output"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  futhark_i32_2d *img = new futhark_i32_2d;
  img->shape[0] = h; img->shape[1] = w;
  const size_t bytes = (size_t)(h > 0 ? h : 0) * (size_t)(w > 0 ? w : 0) * sizeof(int32_t);
  cudaError_t e = cudaMallocAsync(&img->dev, bytes ? bytes : 4, ctx->stream);
  if (e != cudaSuccess) { set_error(ctx, "render: cudaMallocAsync: %s", cudaGetErrorString(e)); delete img; return 1; }
  if (!ctx->peers.empty()) {  // single-process multi-GPU (RAY_GPUS > 1): api_multigpu.cu
    if (render_multi_device(ctx, img, h, w, spp, p)) { cudaFreeAsync(img->dev, ctx->stream); delete img; return 1; }
    *out0 = img;
    return 0;
  }
  // With a shard configured, the row-major frame only receives this rank's tiles; clear the rest.
  if (ctx->cfg.world > 1) cudaMemsetAsync(img->dev, 0, bytes, ctx->stream);
  Frame f{p, h, w, spp, ctx->cfg.rank, ctx->cfg.world, img->dev};
  if (render_frame(ctx, f)) {
    cudaFreeAsync(img->dev, ctx->stream);
    delete img;
    return 1;
  }
  *out0 = img;
  return 0;
}

int futhark_entry_render(struct futhark_context *ctx, struct futhark_i32_2d **out0, const int64_t h, const int64_t w,
                         const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  return ray_b200_entry_render_spp(ctx, out0, h, w, ctx->cfg.spp, p);
}

int ray_b200_render_into(struct futhark_context *ctx, int32_t *out_pix_dev, float *out_rgb_dev, int64_t h, int64_t w, int32_t spp,
                         const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out_pix_dev) { set_error(ctx, "render_into: out_pix_dev is required"); return 1; }
  if (!ctx->peers.empty()) { set_error(ctx, "render_into: not available on a single-process multi-GPU context (RAY_GPUS > 1): only futhark_entry_render / ray_b200_entry_render_spp gather the helper devices' tiles"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, spp, ctx->cfg.rank, ctx->cfg.world, out_pix_dev, out_rgb_dev};
  return render_frame(ctx, f);
}

int ray_b200_render_accumulate(struct futhark_context *ctx, float *accum_dev, int64_t h, int64_t w, int32_t s_begin,
                               int32_t s_end, int32_t *out_pix_dev, float *out_rgb_dev,
                               const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!ctx->peers.empty()) { set_error(ctx, "render_accumulate: not available on a single-process multi-GPU context (RAY_GPUS > 1)"); return 1; }
  if (s_begin < 0 || s_end <= s_begin) { set_error(ctx, "render_accumulate: bad sample range [%d, %d)", s_begin, s_end); return 1; }
  if (!accum_dev) { set_error(ctx, "render_accumulate: accum_dev is required"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, s_end - s_begin, ctx->cfg.rank, ctx->cfg.world, out_pix_dev, out_rgb_dev};
  f.kind = Query::kAccumulate;
  f.q.accum = accum_dev;
  f.q.s_begin = s_begin;
  return render_frame(ctx, f);
}

}  // extern "C"

// ray_b200_render_adaptive (m2_dev == NULL, Query::kAdaptive) and ray_b200_render_adaptive_var (Query::kAdaptiveVar),
// whose errors carry the name `what`
static int render_adaptive(struct futhark_context *ctx, float *accum_dev, float *m2_dev, int32_t *counts_dev,
                           const uint8_t *mask_dev, int64_t h, int64_t w, int32_t n_add, int32_t *out_pix_dev,
                           float *out_rgb_dev, const struct futhark_opaque_prepared_scene *p, bool var, const char *what) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!ctx->peers.empty()) { set_error(ctx, "%s: not available on a single-process multi-GPU context (RAY_GPUS > 1)", what); return 1; }
  if (ctx->cfg.world > 1) { set_error(ctx, "%s: not available with a shard set (rank %d of %d)", what, ctx->cfg.rank, ctx->cfg.world); return 1; }
  if (n_add < 1) { set_error(ctx, "%s: n_add must be >= 1, got %d", what, n_add); return 1; }
  if (!accum_dev) { set_error(ctx, "%s: accum_dev is required", what); return 1; }
  if (var && !m2_dev) { set_error(ctx, "%s: m2_dev is required", what); return 1; }
  if (!counts_dev) { set_error(ctx, "%s: counts_dev is required", what); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, n_add, 0, 1, out_pix_dev, out_rgb_dev};
  f.kind = var ? Query::kAdaptiveVar : Query::kAdaptive;
  f.q.accum = accum_dev;
  f.q.m2 = m2_dev;
  f.q.sample_counts = counts_dev;
  f.q.mask = mask_dev;
  RenderParams P;
  LaunchConfig lc;
  if (fill_params(ctx, f, P, lc)) return 1;
  // The selection list, one item per pixel at most, and its counter in front of it: stream-ordered memory, freed behind the
  // launch, so nothing is held between calls
  int32_t *sel = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&sel, ((size_t)P.local_tiles * kTilePixels + 1) * sizeof(int32_t), ctx->stream));
  f.q.n_sel = sel;
  f.q.sel = sel + 1;
  int rc = do_render(ctx, f, P, lc);
  const cudaError_t fe = cudaFreeAsync(sel, ctx->stream);
  if (!rc && fe != cudaSuccess) { set_error(ctx, "%s: %s", what, cudaGetErrorString(fe)); rc = 1; }
  return rc;
}

extern "C" {

int ray_b200_render_adaptive(struct futhark_context *ctx, float *accum_dev, int32_t *counts_dev, const uint8_t *mask_dev,
                             int64_t h, int64_t w, int32_t n_add, int32_t *out_pix_dev, float *out_rgb_dev,
                             const struct futhark_opaque_prepared_scene *p) {
  return render_adaptive(ctx, accum_dev, nullptr, counts_dev, mask_dev, h, w, n_add, out_pix_dev, out_rgb_dev, p, false,
                         "render_adaptive");
}

int ray_b200_render_adaptive_var(struct futhark_context *ctx, float *accum_dev, float *m2_dev, int32_t *counts_dev,
                                 const uint8_t *mask_dev, int64_t h, int64_t w, int32_t n_add, int32_t *out_pix_dev,
                                 float *out_rgb_dev, const struct futhark_opaque_prepared_scene *p) {
  return render_adaptive(ctx, accum_dev, m2_dev, counts_dev, mask_dev, h, w, n_add, out_pix_dev, out_rgb_dev, p, true,
                         "render_adaptive_var");
}

int ray_b200_adaptive_select(struct futhark_context *ctx, const float *accum_dev, const float *m2_dev, const int32_t *counts_dev,
                             int64_t h, int64_t w, float rel_err, float mean_floor, int32_t min_count, int32_t max_count,
                             uint8_t *mask_dev, int32_t *n_selected_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!image_size_ok(h, w)) { set_error(ctx, "adaptive_select: bad image size %lldx%lld", (long long)h, (long long)w); return 1; }
  if (!accum_dev || !m2_dev || !counts_dev || !mask_dev) {
    set_error(ctx, "adaptive_select: accum_dev, m2_dev, counts_dev and mask_dev are required");
    return 1;
  }
  if (!(std::isfinite(rel_err) && rel_err >= 0.0f)) { set_error(ctx, "adaptive_select: rel_err must be finite and >= 0, got %g", (double)rel_err); return 1; }
  if (!(std::isfinite(mean_floor) && mean_floor >= 0.0f)) {
    set_error(ctx, "adaptive_select: mean_floor must be finite and >= 0, got %g", (double)mean_floor);
    return 1;
  }
  if (min_count < 2) { set_error(ctx, "adaptive_select: min_count must be >= 2 (the variance needs two samples), got %d", min_count); return 1; }
  if (max_count < min_count) { set_error(ctx, "adaptive_select: max_count %d is below min_count %d", max_count, min_count); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  if (n_selected_dev) CUDA_TRY(ctx, cudaMemsetAsync(n_selected_dev, 0, sizeof(int32_t), ctx->stream));
  launch_adaptive_error_select(accum_dev, m2_dev, counts_dev, h * w, rel_err, mean_floor, min_count, max_count, mask_dev,
                               n_selected_dev, ctx->stream, &ctx->launches);
  CUDA_TRY(ctx, cudaGetLastError());
  return 0;
}

int ray_b200_render_views_into(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p,
                               const float *cams7_host, int32_t n_views, int64_t h, int64_t w, int32_t spp,
                               int32_t *out_pix_dev, float *out_rgb_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!ctx->peers.empty()) { set_error(ctx, "render_views_into: not available on a single-process multi-GPU context (RAY_GPUS > 1)"); return 1; }
  if (ctx->cfg.world > 1) { set_error(ctx, "render_views_into: not available with a shard set (rank %d of %d)", ctx->cfg.rank, ctx->cfg.world); return 1; }
  if (n_views < 1) { set_error(ctx, "render_views_into: n_views must be >= 1, got %d", n_views); return 1; }
  if (!cams7_host) { set_error(ctx, "render_views_into: cams7_host is required"); return 1; }
  if (!out_pix_dev) { set_error(ctx, "render_views_into: out_pix_dev is required"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, spp, 0, 1, out_pix_dev, out_rgb_dev};
  f.kind = Query::kViews;
  f.q.n_views = n_views;
  RenderParams P;
  LaunchConfig lc;
  if (fill_params(ctx, f, P, lc)) return 1;
  // View v's camera is what prepare_scene(h, w) of a scene with camera cams7[v] makes: make_camera with this call's aspect
  // ratio (ray.fut:243-244).  The table goes to stream-ordered device memory, freed behind the launch, so the caller may
  // reuse cams7_host as soon as the call returns.
  static_assert(sizeof(CameraRec) == 12 * sizeof(float), "a view's camera is RenderParams::cam's 12 floats");
  std::vector<CameraRec> table((size_t)n_views);
  for (size_t v = 0; v < table.size(); v++) {
    HostScene s;
    const float *c = cams7_host + 7 * v;
    memcpy(s.look_from, c, 12); memcpy(s.look_at, c + 3, 12); s.fov = c[6];
    table[v] = make_camera(s, h, w);
  }
  const size_t bytes = table.size() * sizeof(CameraRec);
  float *cams_dev = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&cams_dev, bytes, ctx->stream));
  const cudaError_t ce = cudaMemcpyAsync(cams_dev, table.data(), bytes, cudaMemcpyHostToDevice, ctx->stream);
  f.q.cams = cams_dev;
  int rc = 0;
  if (ce != cudaSuccess) { set_error(ctx, "render_views_into: camera table upload failed: %s", cudaGetErrorString(ce)); rc = 1; }
  if (!rc) rc = do_render(ctx, f, P, lc);
  const cudaError_t fe = cudaFreeAsync(cams_dev, ctx->stream);
  if (!rc && fe != cudaSuccess) { set_error(ctx, "render_views_into: %s", cudaGetErrorString(fe)); rc = 1; }
  return rc;
}

int ray_b200_render_gbuffer(struct futhark_context *ctx, const struct futhark_opaque_prepared_scene *p, int64_t h, int64_t w,
                            int32_t spp, int32_t *id_dev, float *depth_dev, float *normal_dev, float *albedo_dev,
                            int32_t *coverage_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!ctx->peers.empty()) { set_error(ctx, "render_gbuffer: not available on a single-process multi-GPU context (RAY_GPUS > 1)"); return 1; }
  if (ctx->cfg.world > 1) { set_error(ctx, "render_gbuffer: not available with a shard set (rank %d of %d)", ctx->cfg.rank, ctx->cfg.world); return 1; }
  if (!id_dev && !depth_dev && !normal_dev && !albedo_dev && !coverage_dev) {
    set_error(ctx, "render_gbuffer: every output is NULL");
    return 1;
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, spp, 0, 1};
  f.kind = Query::kGBuffer;
  f.q.perm = p ? p->dev.perm : nullptr;
  f.q.gb_id = id_dev;
  f.q.gb_depth = depth_dev;
  f.q.gb_normal = normal_dev;
  f.q.gb_albedo = albedo_dev;
  f.q.gb_coverage = coverage_dev;
  return render_frame(ctx, f);
}

int ray_b200_render_host(struct futhark_context *ctx, int32_t *out_pix_host, float *out_rgb_host, int64_t h, int64_t w, int32_t spp,
                         const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out_pix_host) { set_error(ctx, "render_host: out_pix_host is required"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  const size_t px = (size_t)h * (size_t)w;
  int32_t *d_pix = nullptr;
  float *d_rgb = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&d_pix, px * 4, ctx->stream));
  if (out_rgb_host) CUDA_TRY(ctx, cudaMallocAsync(&d_rgb, px * 12, ctx->stream));
  Frame f{p, h, w, spp, 0, 1, d_pix, d_rgb};
  int rc = render_frame(ctx, f);
  if (!rc) {
    if (cudaMemcpyAsync(out_pix_host, d_pix, px * 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) rc = 1;
    if (!rc && d_rgb && cudaMemcpyAsync(out_rgb_host, d_rgb, px * 12, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) rc = 1;
    if (rc) set_error(ctx, "render_host: device-to-host copy failed");
  }
  cudaFreeAsync(d_pix, ctx->stream);
  if (d_rgb) cudaFreeAsync(d_rgb, ctx->stream);
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess && !rc) { set_error(ctx, "render_host: kernel failed: %s", cudaGetErrorString(cudaGetLastError())); rc = 1; }
  return rc;
}

int64_t ray_b200_shard_tiles(int64_t h, int64_t w, int32_t rank, int32_t world) {
  if (world < 1 || rank < 0 || rank >= world || h <= 0 || w <= 0) return -1;
  return tiles_of_rank(h, w, rank, world);
}
int64_t ray_b200_shard_tiles_padded(int64_t h, int64_t w, int32_t world) {
  if (world < 1 || h <= 0 || w <= 0) return -1;
  return (tiles_total(h, w) + world - 1) / world;
}
int ray_b200_render_shard_into(struct futhark_context *ctx, int32_t *out_tiles_dev, int64_t h, int64_t w, int32_t spp,
                               const struct futhark_opaque_prepared_scene *p) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out_tiles_dev) { set_error(ctx, "render_shard_into: null output"); return 1; }
  if (!ctx->peers.empty()) { set_error(ctx, "render_shard_into: not available on a single-process multi-GPU context (RAY_GPUS > 1)"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  Frame f{p, h, w, spp, ctx->cfg.rank, ctx->cfg.world, out_tiles_dev, nullptr, true};
  return render_frame(ctx, f);
}
// Several frames in one call, up to two of them in flight: job i runs on lane i % 2, lane 1 forks from the context's
// stream at the start of the call and joins it at the end, so for the caller the batch behaves like one stream-ordered
// operation.  Why: a frame ends on its longest paths (a 50-bounce path is ~50 dependent traversals) while most SMs are
// already idle; the persistent kernel of the NEXT frame cannot start there before the stream order lets it.  With the
// second lane its CTAs take over every SM the moment the previous frame's CTA retires.
int ray_b200_render_batch(struct futhark_context *ctx, const struct ray_b200_render_job *jobs, int32_t n) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (n < 0 || (n > 0 && !jobs)) { set_error(ctx, "render_batch: bad arguments"); return 1; }
  if (n == 0) return 0;
  if (!ctx->peers.empty()) { set_error(ctx, "render_batch: not available on a single-process multi-GPU context (RAY_GPUS > 1)"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  for (int32_t i = 0; i < n; i++) {
    if (!jobs[i].out_dev) { set_error(ctx, "render_batch: job %d has no output buffer", i); return 1; }
    if (jobs[i].shard_layout && jobs[i].out_rgb_dev) { set_error(ctx, "render_batch: job %d: no float output in the shard layout", i); return 1; }
  }
  // the wavefront kernel's ray queues and the warp trace exist once per context: those batches run in order on lane 0
  const bool lanes_ok = !kernel_info(resolve_kernel(ctx, Query::kPixels, 1)).wavefront_queues && !ctx->warp_trace;
  const bool pipe = ctx->pipeline && lanes_ok;   // frames alternate lanes across calls, no join at the end
  const bool two_lanes = lanes_ok && (n > 1 || pipe);
  futhark_context::Lane &L1 = ctx->lanes[1];
  if (two_lanes && !L1.stream) {
    CUDA_TRY(ctx, cudaStreamCreateWithFlags(&L1.stream, cudaStreamNonBlocking));
    CUDA_TRY(ctx, cudaMalloc(&L1.work_cursor, 64));
  }
  CUDA_TRY(ctx, cudaEventRecord(ctx->ev_start, ctx->stream));
  if (two_lanes) {
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(L1.stream, ctx->ev_fork, 0));
  }
  int rc = 0;
  for (int32_t i = 0; i < n && !rc; i++) {
    const ray_b200_render_job &j = jobs[i];
    const int lane = pipe ? (int)(ctx->lane_seq++ & 1u) : (two_lanes ? (i & 1) : 0);
    // (a shard-layout job has no float output: checked above)
    Frame f{j.prepared, j.h, j.w, j.spp > 0 ? j.spp : ctx->cfg.spp, ctx->cfg.rank, ctx->cfg.world, j.out_dev, j.out_rgb_dev, j.shard_layout != 0};
    FrameFlags ff{j.wait_flag, j.wait_value, j.done_flag};
    rc = render_frame(ctx, f, lane, false, (ff.wait_flag || ff.done_flag) ? &ff : nullptr);
  }
  // join even after a failure: whatever was enqueued on lane 1 must be ordered before later work on the context's stream
  // (pipelined submission: no join - the caller orders its reads, see ray_b200_context_set_pipeline)
  if (two_lanes && (!pipe || rc)) {
    if (cudaEventRecord(ctx->ev_join, L1.stream) != cudaSuccess || cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0) != cudaSuccess) {
      if (!rc) set_error(ctx, "render_batch: join failed");
      rc = 1;
    }
  }
  if (!rc) {
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_stop, ctx->stream));
    ctx->have_timing = true;
  }
  return rc;
}

int64_t ray_b200_render_job_size(void) { return (int64_t)sizeof(struct ray_b200_render_job); }

int ray_b200_context_last_plan(struct futhark_context *ctx, struct ray_b200_plan *out) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out) { set_error(ctx, "context_last_plan: null output"); return 1; }
  *out = ctx->last_plan;
  return 0;
}
int64_t ray_b200_plan_size(void) { return (int64_t)sizeof(struct ray_b200_plan); }

int ray_b200_context_set_pipeline(struct futhark_context *ctx, int32_t on) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  if (ctx->pipeline && !on && ctx->lanes[1].stream) {  // leaving the mode: everything in flight joins the context's stream
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->lanes[1].stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  }
  ctx->pipeline = on != 0;
  return 0;
}
int ray_b200_pipeline_join(struct futhark_context *ctx) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  if (ctx->lanes[1].stream) {
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->lanes[1].stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  }
  return 0;
}

int ray_b200_detile(struct futhark_context *ctx, const int32_t *gathered_dev, int32_t *out_pix_dev, int64_t h, int64_t w, int32_t world) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!gathered_dev || !out_pix_dev || world < 1 || h <= 0 || w <= 0) { set_error(ctx, "detile: bad argument"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  launch_detile(gathered_dev, out_pix_dev, h, w, world, ray_b200_shard_tiles_padded(h, w, world), ctx->stream, &ctx->launches);
  CUDA_TRY(ctx, cudaGetLastError());
  return 0;
}

// ---- peer-memory frames (include/ray_b200.h) ----
int ray_b200_ipc_alloc(struct futhark_context *ctx, int64_t bytes, void **dev_ptr, unsigned char *handle64) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!dev_ptr || !handle64 || bytes <= 0) { set_error(ctx, "ipc_alloc: bad argument"); return 1; }
  static_assert(sizeof(cudaIpcMemHandle_t) == RAY_B200_IPC_HANDLE_BYTES, "IPC handle size");
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  void *p = nullptr;
  CUDA_TRY(ctx, cudaMalloc(&p, (size_t)bytes));   // plain cudaMalloc: memory of the stream-ordered pool cannot be exported
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaMemset(p, 0, (size_t)bytes);
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); set_error(ctx, "ipc_alloc: %s", cudaGetErrorString(e)); return 1; }
  memcpy(handle64, &h, sizeof h);
  *dev_ptr = p;
  return 0;
}
int ray_b200_ipc_free(struct futhark_context *ctx, void *dev_ptr) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  if (dev_ptr) CUDA_TRY(ctx, cudaFree(dev_ptr));
  return 0;
}
int ray_b200_ipc_open(struct futhark_context *ctx, const unsigned char *handle64, void **dev_ptr) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!dev_ptr || !handle64) { set_error(ctx, "ipc_open: bad argument"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof h);
  CUDA_TRY(ctx, cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));  // maps the peer GPU's memory (NVLink P2P)
  return 0;
}
int ray_b200_ipc_close(struct futhark_context *ctx, void *dev_ptr) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  if (dev_ptr) CUDA_TRY(ctx, cudaIpcCloseMemHandle(dev_ptr));
  return 0;
}
int ray_b200_flag_wait(struct futhark_context *ctx, void *stream, uint32_t *flag_dev, uint32_t value, int32_t timeout_ms) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!flag_dev) { set_error(ctx, "flag_wait: null flag"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  launch_flag_wait(flag_dev, value, (long long)timeout_ms * 1000000ll, ctx->flag_timeouts, stream ? (cudaStream_t)stream : ctx->stream);
  CUDA_TRY(ctx, cudaGetLastError());
  ctx->launches++;
  return 0;
}
int ray_b200_flag_set(struct futhark_context *ctx, void *stream, uint32_t *flag_dev, uint32_t value) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!flag_dev) { set_error(ctx, "flag_set: null flag"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  launch_flag_set(flag_dev, value, stream ? (cudaStream_t)stream : ctx->stream);
  CUDA_TRY(ctx, cudaGetLastError());
  ctx->launches++;
  return 0;
}
int ray_b200_flag_status(struct futhark_context *ctx, int64_t *timeouts) {
  if (bad_ctx(ctx) || !timeouts) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  unsigned long long v = 0;
  CUDA_TRY(ctx, cudaMemcpy(&v, ctx->flag_timeouts, sizeof v, cudaMemcpyDeviceToHost));
  *timeouts = (int64_t)v;
  return 0;
}
int ray_b200_copy_to_host_async(struct futhark_context *ctx, void *stream, void *host_dst, const void *dev_src, int64_t bytes) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!host_dst || !dev_src || bytes < 0) { set_error(ctx, "copy_to_host_async: bad argument"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  CUDA_TRY(ctx, cudaMemcpyAsync(host_dst, dev_src, (size_t)bytes, cudaMemcpyDeviceToHost, stream ? (cudaStream_t)stream : ctx->stream));
  return 0;
}

int ray_b200_count_work(struct futhark_context *ctx, int64_t h, int64_t w, int32_t spp, const struct futhark_opaque_prepared_scene *p,
                        struct ray_b200_counters *out) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (!out) { set_error(ctx, "count_work: null output"); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  int32_t *scratch = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync(&scratch, (size_t)h * w * 4, ctx->stream));
  Frame f{p, h, w, spp, 0, 1, scratch};
  RenderParams P;
  LaunchConfig lc;
  int rc = fill_params(ctx, f, P, lc);
  if (!rc) {
    cudaMemsetAsync(ctx->counters, 0, 4 * sizeof(unsigned long long), ctx->stream);
    launch_count_work(P, ctx->stream, &ctx->launches);
    unsigned long long host[4] = {0, 0, 0, 0};
    if (cudaMemcpyAsync(host, ctx->counters, sizeof host, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
      set_error(ctx, "count_work: %s", cudaGetErrorString(cudaGetLastError()));
      rc = 1;
    }
    out->segments = host[0]; out->node_steps = host[1]; out->box_tests = host[2]; out->leaf_tests = host[3];
  }
  cudaFreeAsync(scratch, ctx->stream);
  return rc;
}

}  // extern "C"

extern "C" int ray_b200_render_scene_batch_into(struct futhark_context *ctx, const struct ray_b200_scene_batch *b, int64_t h,
                                                int64_t w, int32_t spp, int32_t *out_pix_dev, float *out_rgb_dev) {
  if (bad_ctx(ctx)) return 1;
  std::lock_guard<std::mutex> g(ctx->mu);
  const char *what = "render_scene_batch_into";
  if (!ctx->peers.empty()) { set_error(ctx, "%s: not available on a single-process multi-GPU context (RAY_GPUS > 1)", what); return 1; }
  if (ctx->cfg.world > 1) { set_error(ctx, "%s: not available with a shard set (rank %d of %d)", what, ctx->cfg.rank, ctx->cfg.world); return 1; }
  if (!b || !b->scene.dev.block) { set_error(ctx, "%s: invalid scene batch", what); return 1; }
  if (!out_pix_dev) { set_error(ctx, "%s: out_pix_dev is required", what); return 1; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
  // one launch over every member's tree: the scene half of the parameters comes from all of them (fill_scene_params over
  // n_inner_of / n_leaves_of), and each member's camera and root box from the batch's device tables
  Frame f{&b->scene, h, w, spp, 0, 1, out_pix_dev, out_rgb_dev};
  f.kind = Query::kSceneBatch;
  f.q.n_views = b->scene.scenes;
  f.q.cams = b->scene.dev.cams;
  f.q.root_boxes = reinterpret_cast<const float *>(b->scene.dev.results);
  f.q.scene_off = b->scene.dev.scene_off;
  return render_frame(ctx, f);
}
