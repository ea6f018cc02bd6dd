#!/usr/bin/env python
"""Ray queries on one GPU (include/ray_b200.h "ray queries"); prints one JSON line.

    python tools/bench_rays.py [--rays N] [--seed S] [--only WORKLOAD,...]

- rays_irreg_paths_4M: N random rays (default 2^22) through trace_paths on irreg;
- rays_irreg_hits_4M: the same rays through trace_hits;
- rays_random1M_hits_4M: N random rays through trace_hits on the 1 M-sphere scene;
- camera_rays_irreg_1000: irreg's 1000x1000 camera rays through trace_paths, next to the render call of the same frame
  (the generic path against the fused one) and whether the quantised colours equal its pixels;
- rays_irreg_occluded_4M, rays_random1M_occluded_4M: the random rays of the hit workloads through trace_occluded with the
  interval (0.1, 1e9);
- shadow_irreg_1000: irreg's 1000x1000 camera rays through trace_hits, then a segment from every hit point to a point
  light above the scene (direction = light - point, interval (1e-4, 1 - 1e-4)) through trace_occluded;
- rays_irreg_multi{1,4,16}_4M, rays_random1M_multi4_4M: the random rays of the hit workloads through trace_multi_hits
  with k = 1, 4, 16 (irreg) and k = 4 (1 M spheres), interval (0.1, 1e9);
- depth_irreg_1000_multi8: irreg's 1000x1000 camera rays through trace_multi_hits with k = 8 and the interval (0, 1e9),
  a depth-complexity query;
- rays_{irreg,random1M}_{hits,occluded,multi4}_ranged_4M: the random rays of the hit workloads, each carrying the interval
  (0.1, 1e9), through the ranged entry points (k = 4), with the per-call entry point on the same rays and interval beside
  it (`percall_ms`): the cost of carrying the interval per ray;
- lights4_irreg_1000: irreg's 1000x1000 camera rays through trace_hits, then from every hit point a shadow ray toward one
  of four lights above the scene, chosen per ray, with a unit direction and the interval (1e-2, distance - 1e-4),
  through trace_occluded_ranged; beside it (`segment_ms`) the same segments in the per-call form (direction = light -
  point, (1e-4, 1 - 1e-4)) through trace_occluded.  The two forms round differently, so each has its own parity.
  In these records both times are the smaller of two medians, the two forms alternated (ranged, per-call, ranged,
  per-call).
An occlusion or multi-hit record has trace_hits' time on the same rays and interval beside its own (`hits_ms`), and the
fraction of rays occluded or the mean count of a multi-hit query; its Mrays/s counts one ray per query.
Random rays come from a fixed seed: origins uniform in the scene's bounding box expanded by 10 % per side, directions
uniform on the sphere, so every run sees the same inputs.  `ms` = the median of 3 queries (CUDA events of the context,
after one warm-up query that loads the kernel); Mrays/s = objs_hit calls / kernel time (one per ray for a hit query, the
segments trace_paths reports for a path query); `parity` = differing values against the CPU oracle
(tests/ray_query_oracle.py; tests/ray_interval_oracle.py for the ranged queries) on 4096 rays spread over the batch.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def random_rays(np, spheres, count, seed):
    lo = (spheres[:, :3] - spheres[:, 6:7]).min(0)
    hi = (spheres[:, :3] + spheres[:, 6:7]).max(0)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo), (count, 3)).astype(np.float32)
    d = rng.standard_normal((count, 3)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([o, d / np.linalg.norm(d, axis=1, keepdims=True)], 1), np.float32)


def ranged_workload(np, torch, R, Q, RQ, ctx, timed, bits, name, n_spheres, hh, ww, sc, pr, mode, k, args):
    """One workload of rays that carry their own interval (struct ray_b200_ray), with the per-call form beside it."""
    o = Q.prepare(name, hh, ww, n=n_spheres)            # the per-call queries
    ro = RQ.prepare(name, hh, ww, n=n_spheres)          # the ranged ones
    if mode == "lights":
        cam = torch.from_numpy(R.camera_rays(pr.info()["camera"], hh, ww).reshape(-1, 6)).cuda()
        hit = ctx.trace_hits(pr, cam)
        p = hit["p"].cpu().numpy()[hit["t"].cpu().numpy() >= 0]
        s = sc.arrays()[0]
        lo, hi = (s[:, :3] - s[:, 6:7]).min(0), (s[:, :3] + s[:, 6:7]).max(0)
        c, ext = (lo + hi) / 2, hi - lo
        lights = np.float32([[c[0] + sx * ext[0] / 4, hi[1] + max(ext[0], ext[2]) / 4, c[2] + sz * ext[2] / 4]
                             for sx in (-1, 1) for sz in (-1, 1)])   # the construction of tests/test_ray_intervals.py
        v = lights[np.random.default_rng(args.seed).integers(0, 4, p.shape[0])] - p
        dist = np.sqrt((v * v).sum(1, dtype=np.float32)).astype(np.float32)
        rays8 = np.concatenate([p, np.full((p.shape[0], 1), 1e-2, np.float32), v / dist[:, None], (dist - np.float32(1e-4))[:, None]], 1)
        rays6 = np.concatenate([p, v], 1)   # the per-call segment form of the same rays
        t_min, t_max = 1e-4, 1 - 1e-4
    else:
        rays6 = random_rays(np, sc.arrays()[0], args.rays, args.seed)
        t_min, t_max = 0.1, 1e9
        rays8 = np.concatenate([rays6[:, :3], np.full((rays6.shape[0], 1), t_min, np.float32), rays6[:, 3:],
                                np.full((rays6.shape[0], 1), t_max, np.float32)], 1)
    rays6, rays8 = np.ascontiguousarray(rays6, np.float32), np.ascontiguousarray(rays8, np.float32)
    cnt = rays8.shape[0]
    d6, d8 = torch.from_numpy(rays6).cuda(), torch.from_numpy(rays8).cuda()
    kk = max(k, 1)
    out6 = torch.empty((cnt, kk, 8), dtype=torch.float32, device="cuda")
    out8 = torch.empty((cnt, kk, 8), dtype=torch.float32, device="cuda")
    c6 = torch.empty((cnt,), dtype=torch.int32, device="cuda")
    c8 = torch.empty((cnt,), dtype=torch.int32, device="cuda")
    occ6 = torch.empty((cnt,), dtype=torch.bool, device="cuda")
    occ8 = torch.empty((cnt,), dtype=torch.bool, device="cuda")
    torch.cuda.synchronize()   # the context's own stream is not ordered after torch's
    if mode == "hits_r":
        ranged_q = lambda: ctx.trace_hits_ranged_into(d8.data_ptr(), cnt, pr, out8.data_ptr())
        per_call = lambda: ctx.trace_hits_into(d6.data_ptr(), cnt, pr, out6.data_ptr(), t_min=t_min, t_max=t_max)
    elif mode == "multi_r":
        ranged_q = lambda: ctx.trace_multi_hits_ranged_into(d8.data_ptr(), cnt, pr, k, out8.data_ptr(), c8.data_ptr())
        per_call = lambda: ctx.trace_multi_hits_into(d6.data_ptr(), cnt, pr, k, out6.data_ptr(), c6.data_ptr(), t_min=t_min, t_max=t_max)
    else:
        ranged_q = lambda: ctx.trace_occluded_ranged_into(d8.data_ptr(), cnt, pr, occ8.data_ptr())
        per_call = lambda: ctx.trace_occluded_into(d6.data_ptr(), cnt, pr, occ6.data_ptr(), t_min=t_min, t_max=t_max)
    # alternated, so that both forms see the same clocks: ranged, per-call, ranged, per-call
    ms, ms_call = timed(ranged_q), timed(per_call)
    ms, ms_call = min(ms, timed(ranged_q)), min(ms_call, timed(per_call))
    rec = {"rays": cnt, "ms": round(ms, 3), "Mrays_s": round(cnt / ms / 1e3, 1)}
    rec["percall_ms" if mode != "lights" else "segment_ms"] = round(ms_call, 3)
    rec["ranged_over_percall" if mode != "lights" else "ranged_over_segment"] = round(ms / ms_call, 3)
    if mode != "lights":
        rec["t_min"], rec["t_max"] = t_min, t_max
    sub = np.linspace(0, cnt - 1, 4096).astype(np.int64)
    if mode == "hits_r":
        rec["parity"] = int((bits(out8[:, 0].cpu().numpy()[sub]) != bits(ro.trace_hits_ranged(rays8[sub]))).sum())
        rec["percall_parity"] = int((bits(out6[:, 0].cpu().numpy()[sub]) != bits(o.trace_hits(rays6[sub], t_min, t_max))).sum())
    elif mode == "multi_r":
        want, want_c = ro.trace_multi_hits_ranged(rays8[sub], k)
        rec["parity"] = int((bits(out8.cpu().numpy()[sub]) != bits(want)).sum()) + int((c8.cpu().numpy()[sub] != want_c).sum())
        want, want_c = o.trace_multi_hits(rays6[sub], k, t_min, t_max)
        rec["percall_parity"] = int((bits(out6.cpu().numpy()[sub]) != bits(want)).sum()) + int((c6.cpu().numpy()[sub] != want_c).sum())
        rec["k"], rec["mean_count"] = k, round(float(c8.double().mean()), 3)
    else:
        occ8, occ6 = occ8.cpu().numpy(), occ6.cpu().numpy()
        rec["parity"] = int((occ8[sub] != ro.trace_occluded_ranged(rays8[sub])).sum())
        rec["percall_parity" if mode != "lights" else "segment_parity"] = int((occ6[sub] != o.trace_occluded(rays6[sub], t_min, t_max)).sum())
        rec["occluded_fraction"] = round(float(occ8.mean()), 4)
        if mode == "lights":
            rec["segment_occluded_fraction"] = round(float(occ6.mean()), 4)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=1 << 22)
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    args = ap.parse_args()
    import numpy as np
    import torch

    import ray_query_oracle as Q
    import ray_interval_oracle as RQ
    import raytracers_b200 as R

    def bits(a):
        return np.ascontiguousarray(a, np.float32).view(np.uint32)

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    ctx = R.Context(device=0)

    def timed(fn):
        fn()   # the first query loads the ray-mode kernel
        torch.cuda.synchronize()
        ms = []
        for _ in range(3):
            fn()
            torch.cuda.synchronize()
            ms.append(ctx.last_render_ms())
        return sorted(ms)[1]

    out = {}
    for tag, name, n_spheres, hh, ww, mode, k in (("rays_irreg_paths_4M", "irreg", None, 1000, 1000, "paths", 0),
                                                  ("rays_irreg_hits_4M", "irreg", None, 1000, 1000, "hits", 0),
                                                  ("rays_random1M_hits_4M", "random", 1000000, 2000, 2000, "hits", 0),
                                                  ("camera_rays_irreg_1000", "irreg", None, 1000, 1000, "camera", 0),
                                                  ("rays_irreg_occluded_4M", "irreg", None, 1000, 1000, "occluded", 0),
                                                  ("rays_random1M_occluded_4M", "random", 1000000, 2000, 2000, "occluded", 0),
                                                  ("shadow_irreg_1000", "irreg", None, 1000, 1000, "shadow", 0),
                                                  ("rays_irreg_multi1_4M", "irreg", None, 1000, 1000, "multi", 1),
                                                  ("rays_irreg_multi4_4M", "irreg", None, 1000, 1000, "multi", 4),
                                                  ("rays_irreg_multi16_4M", "irreg", None, 1000, 1000, "multi", 16),
                                                  ("rays_random1M_multi4_4M", "random", 1000000, 2000, 2000, "multi", 4),
                                                  ("depth_irreg_1000_multi8", "irreg", None, 1000, 1000, "depth", 8),
                                                  ("rays_irreg_hits_ranged_4M", "irreg", None, 1000, 1000, "hits_r", 0),
                                                  ("rays_irreg_occluded_ranged_4M", "irreg", None, 1000, 1000, "occluded_r", 0),
                                                  ("rays_irreg_multi4_ranged_4M", "irreg", None, 1000, 1000, "multi_r", 4),
                                                  ("rays_random1M_hits_ranged_4M", "random", 1000000, 2000, 2000, "hits_r", 0),
                                                  ("rays_random1M_occluded_ranged_4M", "random", 1000000, 2000, 2000, "occluded_r", 0),
                                                  ("rays_random1M_multi4_ranged_4M", "random", 1000000, 2000, 2000, "multi_r", 4),
                                                  ("lights4_irreg_1000", "irreg", None, 1000, 1000, "lights", 0)):
        if args.only and tag not in args.only.split(","):
            continue
        sc = ctx.scene(name, n=n_spheres)
        pr = ctx.prepare_scene(hh, ww, sc)
        t_min, t_max = (1e-4, 1 - 1e-4) if mode == "shadow" else ((0.0, 1e9) if mode == "depth" else (0.1, 1e9))
        if mode in ("hits_r", "occluded_r", "multi_r", "lights"):
            out[tag] = ranged_workload(np, torch, R, Q, RQ, ctx, timed, bits, name, n_spheres, hh, ww, sc, pr, mode, k, args)
            pr.free(); sc.free()
            continue
        if mode in ("camera", "shadow", "depth"):
            rays = R.camera_rays(pr.info()["camera"], hh, ww).reshape(-1, 6)
        else:
            rays = random_rays(np, sc.arrays()[0], args.rays, args.seed)
        if mode == "shadow":   # the same construction as tests/test_occlusion.py
            hit = ctx.trace_hits(pr, torch.from_numpy(rays).cuda())
            p = hit["p"].cpu().numpy()[hit["t"].cpu().numpy() >= 0]
            s = sc.arrays()[0]
            lo, hi = (s[:, :3] - s[:, 6:7]).min(0), (s[:, :3] + s[:, 6:7]).max(0)
            light = np.float32([(lo[0] + hi[0]) / 2, hi[1] + (hi[1] - lo[1]), (lo[2] + hi[2]) / 2])
            rays = np.ascontiguousarray(np.concatenate([p, light[None] - p], 1), np.float32)
        cnt = rays.shape[0]
        d_rays = torch.from_numpy(rays).cuda()
        rgb = torch.empty((cnt, 3), dtype=torch.float32, device="cuda")
        seg = torch.empty((cnt,), dtype=torch.int32, device="cuda")
        hits = torch.empty((cnt, 8), dtype=torch.float32, device="cuda")
        occ = torch.empty((cnt,), dtype=torch.bool, device="cuda")
        multi = torch.empty((cnt, max(k, 1), 8), dtype=torch.float32, device="cuda")
        counts = torch.empty((cnt,), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()   # the context's own stream is not ordered after torch's
        if mode in ("multi", "depth"):
            ms = timed(lambda: ctx.trace_multi_hits_into(d_rays.data_ptr(), cnt, pr, k, multi.data_ptr(), counts.data_ptr(),
                                                         t_min=t_min, t_max=t_max))
            segments = cnt
        elif mode in ("occluded", "shadow"):
            ms = timed(lambda: ctx.trace_occluded_into(d_rays.data_ptr(), cnt, pr, occ.data_ptr(), t_min=t_min, t_max=t_max))
            segments = cnt
        elif mode == "hits":
            ms = timed(lambda: ctx.trace_hits_into(d_rays.data_ptr(), cnt, pr, hits.data_ptr()))
            segments = cnt
        else:
            ms = timed(lambda: ctx.trace_paths_into(d_rays.data_ptr(), cnt, pr, rgb.data_ptr(), seg.data_ptr()))
            segments = int(seg.sum(dtype=torch.int64))
        rec = {"rays": cnt, "ms": round(ms, 3), "segments": segments, "Mrays_s": round(segments / ms / 1e3, 1)}
        if mode in ("occluded", "shadow", "multi", "depth"):   # the closest-hit query on the same rays and interval, timed the same way
            rec["t_min"], rec["t_max"] = t_min, t_max
            rec["hits_ms"] = round(timed(lambda: ctx.trace_hits_into(d_rays.data_ptr(), cnt, pr, hits.data_ptr(), t_min=t_min, t_max=t_max)), 3)
        if mode in ("occluded", "shadow"):
            rec["hits_over_occluded"] = round(rec["hits_ms"] / rec["ms"], 3)
            rec["occluded_fraction"] = round(float(occ.float().mean()), 4)
        if mode in ("multi", "depth"):
            rec["k"] = k
            rec["multi_over_hits"] = round(rec["ms"] / rec["hits_ms"], 3)
            rec["mean_count"] = round(float(counts.double().mean()), 3)
            rec["max_count"] = int(counts.max())
        if mode == "camera":   # the fused path: the render call on the same frame
            fr = torch.empty((hh, ww), dtype=torch.int32, device="cuda")
            rec["render_ms"] = round(timed(lambda: ctx.render_into(fr.data_ptr(), hh, ww, pr, spp=1)), 3)
            q = (np.float32(255.99) * rgb.cpu().numpy()).astype(np.int32)
            rec["quantised_equals_render_pixels"] = bool(((q[:, 0] << 16 | q[:, 1] << 8 | q[:, 2]).reshape(hh, ww) == fr.cpu().numpy()).all())
        sub = np.linspace(0, cnt - 1, 4096).astype(np.int64)
        o = Q.prepare(name, hh, ww, n=n_spheres)
        if mode in ("multi", "depth"):
            want, want_counts = o.trace_multi_hits(rays[sub], k, t_min, t_max)
            rec["parity"] = int((bits(multi.cpu().numpy()[sub]) != bits(want)).sum()) + int((counts.cpu().numpy()[sub] != want_counts).sum())
        elif mode in ("occluded", "shadow"):
            rec["parity"] = int((occ.cpu().numpy()[sub] != o.trace_occluded(rays[sub], t_min, t_max)).sum())
        elif mode == "hits":
            rec["parity"] = int((bits(hits.cpu().numpy()[sub]) != bits(o.trace_hits(rays[sub]))).sum())
        else:
            want_rgb, want_seg = o.trace_paths(rays[sub])
            rec["parity"] = int((bits(rgb.cpu().numpy()[sub]) != bits(want_rgb)).sum()) + int((seg.cpu().numpy()[sub] != want_seg).sum())
        out[tag] = rec
        del d_rays, rgb, seg, hits, occ, multi, counts
        pr.free(); sc.free()
    ctx.close()
    print(json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                      "sm_max_mhz": int(gpu[2]) if len(gpu) > 2 else None, "rays": args.rays, "seed": args.seed, **out}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
