#!/usr/bin/env python
"""Nearest-sphere queries (Context.query_nearest_into, query_scene_batch_nearest_into): the k nearest spheres to each
point with no limit on the distance, against the two things a caller could do without them; prints one JSON line.

    python tools/bench_nearest.py [--steps N] [--warmup W] [--only WORKLOAD,...] [--out PATH]

Workloads:
  graph_*       the k = 8 and k = 16 neighbour graph of a random 2^20-sphere scene: every sphere's own centre queried at
                k + 1, with the queries in caller order (random in space) and in the scene's Morton order (prepared_dump's
                perm);
  sdf_*         2^22 unbounded k = 1 probes (the signed distance of the scene) in the box of irreg and of the random
                2^20-sphere scene;
  batch_*       1024 scenes × 64 points at k = 8: 64 random spheres each (uniform), and 16..256 spheres (ragged).

`ms` is the median over --steps timed calls (after --warmup untimed ones) of the device time of one nearest-sphere call
(CUDA events on the context's stream, torch's current stream here).  `radius_ms` is the same for query_spheres (or its
batch form) at k with one radius chosen after the fact, the largest k-th distance of the answer, so that every ball holds
at least k spheres: the best a caller could do with a fixed radius, and `radius_matches` whether its records equal the
nearest-sphere query's bit for bit (the identity of the header).  `brute_ms` is the median device time of a chunked torch
brute force (cdist - rho, then topk) on `brute_queries` of the points, `brute_ms_all_est` that scaled to all of them.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return round(statistics.median(out), 4)


def brute(torch, spheres, pts, k, chunk_elems=1 << 28):
    """(d, idx) [q, k] of the k nearest spheres by d = |c - p| - rho (cdist, then topk), chunked over the points"""
    p, rho = spheres[:, :3], spheres[:, 6]
    step = max(1, chunk_elems // spheres.shape[0])
    ds, idx = [], []
    for a in range(0, pts.shape[0], step):
        d = torch.cdist(pts[a:a + step, :3], p) - rho[None, :]
        t = torch.topk(d, k, dim=1, largest=False)
        ds.append(t.values)
        idx.append(t.indices)
    return torch.cat(ds), torch.cat(idx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    dev = torch.device("cuda", 0)
    ctx = R.Context(device=0)
    ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream)
    rng = np.random.default_rng(1)
    result = {"gpu": gpu[0], "power_limit_w": float(gpu[1]), "max_sm_clock_mhz": float(gpu[2]), "steps": args.steps,
              "warmup": args.warmup, "workloads": {}}
    cam = np.float32([0, 0, 1, 0, 0, 0, 40])

    def want(key):
        return not only or any(key.startswith(o) for o in only)

    def single(key, pr, s_t, balls, k, brute_q, extra=None):
        """balls: [n, 4] with r = +inf; the nearest query at k, query_spheres at k with the radius that holds k for every
        ball, and the torch brute force on the first brute_q balls"""
        n = balls.shape[0]
        near = torch.empty((n, k, 2), dtype=torch.float32, device=dev)
        launches = ctx.launch_count()
        ctx.query_nearest_into(balls.data_ptr(), n, pr, k, near.data_ptr())
        per_call = ctx.launch_count() - launches
        ms = timed(torch, lambda: ctx.query_nearest_into(balls.data_ptr(), n, pr, k, near.data_ptr()), args.steps, args.warmup)
        r_fix = float(near[:, k - 1, 0].max())
        fixed = balls.clone()
        fixed[:, 3] = r_fix
        near_r = torch.empty_like(near)
        cnt = torch.empty((n,), dtype=torch.int32, device=dev)
        rms = timed(torch, lambda: ctx.query_spheres_into(fixed.data_ptr(), n, pr, k, near_r.data_ptr(), cnt.data_ptr()),
                    args.steps, args.warmup)
        row = {"spheres": int(s_t.shape[0]), "queries": n, "k": k, "stale_nodes": pr.info()["stale_nodes"],
               "launches_per_call": per_call, "ms": ms, "queries_per_s": round(n / ms * 1e3),
               "radius": r_fix, "radius_ms": rms, "radius_mean_count": round(float(cnt.double().mean()), 1),
               "radius_matches": bool(torch.equal(near.view(torch.int32), near_r.view(torch.int32))),
               "speedup_vs_radius": round(rms / ms, 2)}
        row.update(extra or {})
        try:
            sub = balls[:brute_q]
            bms = timed(torch, lambda: brute(torch, s_t, sub, k), max(1, args.steps // 2), 1)
            _, bi = brute(torch, s_t, sub, k)
            row.update(brute_queries=brute_q, brute_ms=bms, brute_ms_all_est=round(bms * n / brute_q, 1),
                       brute_nearest_mismatch=int((bi[:, 0] != near[:brute_q, 0, 1].view(torch.int32)).sum()))
            row["speedup_vs_brute"] = round(row["brute_ms_all_est"] / ms, 1)
        except torch.cuda.OutOfMemoryError:
            row["brute_ms"] = "out of memory"
        torch.cuda.empty_cache()
        result["workloads"][key] = row
        print(key, row, file=sys.stderr, flush=True)

    def unbounded(xyz):
        return torch.cat([xyz, torch.full_like(xyz[:, :1], float("inf"))], 1).contiguous()

    big, _ = R.host_scene("random", 1 << 20, 1)
    big_t = torch.from_numpy(big).to(dev)
    # 1. the neighbour graph, in caller order and in Morton order
    if want("graph"):
        pr = ctx.prepare_scene_device(64, 64, big_t, cam)
        perm = torch.from_numpy(pr.dump()["perm"].astype(np.int64)).to(dev)
        for order in ("caller", "morton"):
            xyz = big_t[:, :3] if order == "caller" else big_t[perm, :3]
            balls = unbounded(xyz)
            for k in (8, 16):
                single(f"graph_2p20_k{k}_{order}", pr, big_t, balls, k + 1, 1 << 14, {"neighbours": k, "order": order})
        pr.free()
    # 2. the signed distance at 2^22 probes
    irreg, _ = R.host_scene("irreg")
    for name, s in (("irreg", irreg), ("random2p20", big)):
        key = f"sdf_{name}_k1"
        if not want(key):
            continue
        s_t = torch.from_numpy(s).to(dev)
        pr = ctx.prepare_scene_device(64, 64, s_t, cam)
        lo, hi = s[:, :3].min(0), s[:, :3].max(0)
        pts = torch.from_numpy(rng.uniform(lo, hi, (1 << 22, 3)).astype(np.float32)).to(dev)
        single(key, pr, s_t, unbounded(pts), 1, (1 << 20) if name == "irreg" else 1 << 14)
        pr.free()
    # 3. batches
    for kind in ("uniform", "ragged"):
        key = f"batch_{kind}_1024_m64_k8"
        if not want(key):
            continue
        counts = np.full(1024, 64) if kind == "uniform" else np.random.default_rng(7).integers(16, 257, 1024)
        parts = [R.host_scene("random", int(c), 100 + b)[0] for b, c in enumerate(counts)]
        cams = np.tile(np.float32([0, 0, 1100, 0, 0, 0, 40]), (1024, 1))
        recs = torch.from_numpy(np.concatenate(parts)).to(dev)
        batch = (ctx.prepare_scene_batch(64, 64, recs.view(1024, 64, 7), cams) if kind == "uniform"
                 else ctx.prepare_scene_batch(64, 64, recs, cams, counts=counts))
        pts = np.stack([p[rng.integers(0, len(p), 64), :3] + rng.uniform(-30, 30, (64, 3)) for p in parts]).astype(np.float32)
        balls = torch.from_numpy(np.concatenate([pts, np.full((1024, 64, 1), np.inf, np.float32)], -1)).to(dev)
        near = torch.empty((1024, 64, 8, 2), dtype=torch.float32, device=dev)
        ms = timed(torch, lambda: ctx.query_scene_batch_nearest_into(balls.data_ptr(), 64, batch, 8, near.data_ptr()),
                   args.steps, args.warmup)
        r_fix = float(near[..., 7, 0].max())
        fixed = balls.clone()
        fixed[..., 3] = r_fix
        near_r = torch.empty_like(near)
        cnt = torch.empty((1024, 64), dtype=torch.int32, device=dev)
        rms = timed(torch, lambda: ctx.query_scene_batch_spheres_into(fixed.data_ptr(), 64, batch, 8, near_r.data_ptr(),
                                                                      cnt.data_ptr()), args.steps, args.warmup)
        sub = 64   # the per-scene torch loop on the first 64 scenes, scaled to 1024

        def per_scene():
            off = 0
            for b, p in enumerate(parts[:sub]):
                brute(torch, recs[off:off + len(p)], balls[b], 8)
                off += len(p)
        bms = timed(torch, per_scene, max(1, args.steps // 2), 1)
        row = {"scenes": 1024, "spheres": int(sum(counts)), "points_per_scene": 64, "k": 8, "ms": ms, "radius": r_fix,
               "radius_ms": rms, "radius_mean_count": round(float(cnt.double().mean()), 1),
               "radius_matches": bool(torch.equal(near.view(torch.int32), near_r.view(torch.int32))),
               "speedup_vs_radius": round(rms / ms, 2), "brute_scenes": sub, "brute_ms": bms,
               "brute_ms_all_est": round(bms * 1024 / sub, 1)}
        row["speedup_vs_brute"] = round(row["brute_ms_all_est"] / ms, 1)
        result["workloads"][key] = row
        print(key, row, file=sys.stderr, flush=True)
        batch.free()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
