// C ABI, part 4: the single-process multi-GPU mode (RAY_GPUS = N > 1) — the drop-in multi-GPU path of the unmodified
// futhark/main.c, which knows nothing about ranks.  The context owns one helper context per extra device;
// prepare_scene replicates the LBVH build on every device (api_scene.cu), futhark_entry_render launches every device's
// shard on its own stream, device 0 pulls the shards with cudaMemcpyPeerAsync over NVLink and de-tiles.  (The
// one-process-per-GPU path with torch.distributed is raytracers_b200/distributed.py: NCCL gather, or peer-memory frames.)
#include "api_internal.h"

using namespace rayb200_api;

namespace rayb200_api {

// Helper contexts on devices device+1 .. device+gpus-1, peer access enabled both ways.  On failure the context is
// marked unusable and the error message says why.
int create_helper_contexts(futhark_context *ctx, const futhark_context_config *cfg, int ndev) {
  (void)cfg;
  if (ctx->cfg.device + ctx->cfg.gpus > ndev) {
    ctx->ok = false;
    set_error(ctx, "futhark_context_new: RAY_GPUS=%d needs devices %d..%d but only %d are visible", ctx->cfg.gpus, ctx->cfg.device,
              ctx->cfg.device + ctx->cfg.gpus - 1, ndev);
    return 1;
  }
  for (int r = 1; r < ctx->cfg.gpus; r++) {
    futhark_context_config pc = ctx->cfg;
    pc.device = ctx->cfg.device + r;
    pc.rank = r; pc.world = ctx->cfg.gpus;
    pc.gpus = -1;  // marks a helper: no recursion, no environment override of the device
    futhark_context *peer = futhark_context_new(&pc);
    if (!peer || !peer->ok) {
      char *pe = peer ? futhark_context_get_error(peer) : nullptr;
      ctx->ok = false;
      set_error(ctx, "futhark_context_new: helper context on device %d failed: %s", pc.device, pe ? pe : "?");
      free(pe);
      if (peer) futhark_context_free(peer);
      return 1;
    }
    peer->is_peer = true;
    cudaSetDevice(pc.device);
    cudaEventCreateWithFlags(&peer->peer_done, cudaEventDisableTiming);
    cudaDeviceEnablePeerAccess(ctx->cfg.device, 0);
    cudaSetDevice(ctx->cfg.device);
    cudaDeviceEnablePeerAccess(pc.device, 0);
    cudaGetLastError();  // "already enabled" is fine
    ctx->peers.push_back(peer);
  }
  ctx->cfg.rank = 0; ctx->cfg.world = ctx->cfg.gpus;
  cudaSetDevice(ctx->cfg.device);
  return 0;
}

// One frame on all devices into img->dev (allocated by the caller on device 0's stream; the caller frees it on failure).
// Every device renders its tiles into a compact buffer, device 0 pulls them over NVLink (peer copies ordered by events)
// and de-tiles — the same data flow as the one-process-per-GPU NCCL path, with cudaMemcpyPeerAsync in place of the gather.
int render_multi_device(futhark_context *ctx, futhark_i32_2d *img, int64_t h, int64_t w, int32_t spp, const futhark_opaque_prepared_scene *p) {
  const int world = (int)ctx->peers.size() + 1;
  const int64_t padded = ray_b200_shard_tiles_padded(h, w, world);
  const size_t shard_bytes = (size_t)padded * kTilePixels * sizeof(int32_t);
  auto fail = [&](const char *what) { cudaSetDevice(ctx->cfg.device); set_error(ctx, "render (multi-GPU): %s", what); return 1; };
  if (!p) return fail("invalid prepared scene");
  if (padded < 0) return fail("bad image size");
  if (p->peer_prepared.size() != ctx->peers.size()) return fail("prepared scene was not prepared by this context");
  if (ctx->gathered_bytes < shard_bytes * world) {
    cudaStreamSynchronize(ctx->stream);
    if (ctx->gathered) cudaFree(ctx->gathered);
    ctx->gathered = nullptr; ctx->gathered_bytes = 0;
    if (cudaMalloc(&ctx->gathered, shard_bytes * world) != cudaSuccess) return fail("out of device memory");
    ctx->gathered_bytes = shard_bytes * world;
  }
  for (int r = 1; r < world; r++) {
    futhark_context *peer = ctx->peers[(size_t)r - 1];
    cudaSetDevice(peer->cfg.device);
    if (peer->peer_tiles_bytes < shard_bytes) {
      cudaStreamSynchronize(peer->stream);
      if (peer->peer_tiles) cudaFree(peer->peer_tiles);
      peer->peer_tiles = nullptr; peer->peer_tiles_bytes = 0;
      if (cudaMalloc(&peer->peer_tiles, shard_bytes) != cudaSuccess) return fail("out of device memory on a helper device");
      peer->peer_tiles_bytes = shard_bytes;
    }
    // the previous frame's peer copy out of peer_tiles (on device 0's stream) must have finished before this helper
    // renders into it again: entries are asynchronous, a caller may issue two renders without a sync in between
    if (ctx->gather_pending) cudaStreamWaitEvent(peer->stream, ctx->ev_gathered, 0);
    if (ray_b200_render_shard_into(peer, peer->peer_tiles, h, w, spp, p->peer_prepared[(size_t)r - 1])) {
      char *pe = futhark_context_get_error(peer);
      cudaSetDevice(ctx->cfg.device);
      set_error(ctx, "render on helper device %d: %s", peer->cfg.device, pe ? pe : "?");
      free(pe);
      return 1;
    }
    cudaEventRecord(peer->peer_done, peer->stream);
  }
  cudaSetDevice(ctx->cfg.device);
  // rank 0's own shard straight into slot 0 of the gather buffer
  RenderParams P;
  LaunchConfig lc;
  if (fill_params(ctx, p, h, w, spp, 0, world, ctx->gathered, nullptr, true, P, lc)) return 1;
  if (P.local_tiles < padded)
    cudaMemsetAsync(ctx->gathered + P.local_tiles * kTilePixels, 0, (size_t)(padded - P.local_tiles) * kTilePixels * 4, ctx->stream);
  if (do_render(ctx, P, lc, 0, true, nullptr, p)) return 1;
  for (int r = 1; r < world; r++) {
    futhark_context *peer = ctx->peers[(size_t)r - 1];
    cudaStreamWaitEvent(ctx->stream, peer->peer_done, 0);
    cudaMemcpyPeerAsync(ctx->gathered + (size_t)r * padded * kTilePixels, ctx->cfg.device, peer->peer_tiles, peer->cfg.device, shard_bytes, ctx->stream);
  }
  if (!ctx->ev_gathered) cudaEventCreateWithFlags(&ctx->ev_gathered, cudaEventDisableTiming);
  cudaEventRecord(ctx->ev_gathered, ctx->stream);  // every helper's tile buffer has been read
  ctx->gather_pending = true;
  launch_detile(ctx->gathered, img->dev, h, w, world, padded, ctx->stream, &ctx->launches);
  if (cudaGetLastError() != cudaSuccess) return fail("de-tiling launch failed");
  return 0;
}

}  // namespace rayb200_api
