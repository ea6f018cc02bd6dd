#!/usr/bin/env python
"""Proximity queries (Context.query_spheres, query_scene_batch_spheres): the spheres within a radius of each ball,
nearest first, against a brute force in torch (cdist and topk, chunked); prints one JSON line.

    python tools/bench_proximity.py [--steps N] [--warmup W] [--only WORKLOAD,...] [--out PATH]

Workloads:
  self_2p20     a random 2^20-sphere scene queried with every sphere's own (centre, radius): counts and k = 16;
  probe_*       2^22 random points in the box of irreg and of a random 2^20-sphere scene, r = 1 % of the box's diagonal
                (irreg: 2 %), at k = 1, 8, 64 and count-only (k = 0);
  batch_*       1024 scenes of 64 random spheres with 64 balls each (uniform), and 1024 scenes of 16..256 (ragged);
  refit_*       the complete-box refit of a scene with stale boxes (rgbbox; a 2^20-sphere scene of coincident groups and
                random filler), against the query kernel itself, from torch.profiler kernel times.

`ms` is the median over --steps timed calls (after --warmup untimed ones) of the device time of one call (CUDA events on
the context's stream, torch's current stream here).  `brute_ms` is the median device time of the torch brute force on
`brute_queries` of the balls (all of them where that fits; the self-overlap step is timed on its first 2^16 balls only,
so `brute_ms_all_est` scales it to all of them), and `brute_match` whether its counts and nearest sphere equal the
library's on those balls (the brute force computes distances in its own order, so only sets far from the boundary are
expected to agree: `brute_count_mismatch` counts the balls whose counts differ).  The card's name and power limit are
read in the same run.
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


def brute(torch, spheres, balls, k, chunk_elems=1 << 30):
    """counts [q] and, for k > 0, the k nearest sphere indices [q, k] by d = |c - p| - rho (cdist, then topk)"""
    p, rho = spheres[:, :3], spheres[:, 6]
    step = max(1, chunk_elems // spheres.shape[0])
    counts, idx = [], []
    for a in range(0, balls.shape[0], step):
        b = balls[a:a + step]
        d = torch.cdist(b[:, :3], p) - rho[None, :]
        within = d <= b[:, 3:4]
        counts.append(within.sum(1, dtype=torch.int32))
        if k:
            idx.append(torch.topk(torch.where(within, d, torch.inf), k, dim=1, largest=False).indices)
    return torch.cat(counts), (torch.cat(idx) if k else None)


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

    def want(key):
        return not only or any(key.startswith(o) for o in only)

    def single(key, s, balls, k, brute_q=None):
        pr = ctx.prepare_scene_device(64, 64, s, np.float32([0, 0, 1, 0, 0, 0, 40]))
        n = balls.shape[0]
        near = torch.empty((n, max(k, 1), 2), dtype=torch.float32, device=dev)
        cnt = torch.empty((n,), dtype=torch.int32, device=dev)
        launches = ctx.launch_count()
        ctx.query_spheres_into(balls.data_ptr(), n, pr, k, near.data_ptr() if k else None, cnt.data_ptr())
        per_call = ctx.launch_count() - launches
        ms = timed(torch, lambda: ctx.query_spheres_into(balls.data_ptr(), n, pr, k, near.data_ptr() if k else None,
                                                         cnt.data_ptr()), args.steps, args.warmup)
        row = {"spheres": int(s.shape[0]), "balls": n, "k": k, "stale_nodes": pr.info()["stale_nodes"], "launches_per_call": per_call,
               "ms": ms, "balls_per_s": round(n / ms * 1e3), "mean_count": round(float(cnt.double().mean()), 3),
               "max_count": int(cnt.max())}
        bq = n if brute_q is None else brute_q
        try:
            sub = balls[:bq]
            bms = timed(torch, lambda: brute(torch, s, sub, k), max(1, args.steps // 2), 1)
            bc, bi = brute(torch, s, sub, k)
            row.update(brute_queries=bq, brute_ms=bms, brute_count_mismatch=int((bc != cnt[:bq]).sum()))
            if bq != n:
                row["brute_ms_all_est"] = round(bms * n / bq, 1)
            if k:
                first = near[:bq, 0, 1].view(torch.int32)
                has = bc > 0
                row["brute_nearest_mismatch"] = int((bi[:, 0][has] != first[has]).sum())
            row["speedup_vs_brute"] = round((row.get("brute_ms_all_est") or bms) / ms, 1)
        except torch.cuda.OutOfMemoryError:
            row["brute_ms"] = "out of memory"
        torch.cuda.empty_cache()
        result["workloads"][key] = row
        print(key, row, file=sys.stderr, flush=True)
        pr.free()

    # 1. self-overlap step
    big, _ = R.host_scene("random", 1 << 20, 1)
    big_t = torch.from_numpy(big).to(dev)
    if want("self_2p20"):
        own = big_t[:, [0, 1, 2, 6]].contiguous()
        single("self_2p20_k16", big_t, own, 16, brute_q=1 << 16)
        single("self_2p20_k0", big_t, own, 0, brute_q=1 << 16)
    # 2. probe points
    irreg, _ = R.host_scene("irreg")
    for name, s, frac in (("irreg", irreg, 0.02), ("random2p20", big, 0.01)):
        lo, hi = s[:, :3].min(0), s[:, :3].max(0)
        pts = np.empty((1 << 22, 4), np.float32)
        pts[:, :3] = rng.uniform(lo, hi, (1 << 22, 3))
        pts[:, 3] = frac * float(np.linalg.norm(hi - lo))
        pts_t = torch.from_numpy(pts).to(dev)
        s_t = torch.from_numpy(s).to(dev)
        for k in (0, 1, 8, 64):
            key = f"probe_{name}_k{k}"
            if want(key):
                single(key, s_t, pts_t, k, brute_q=(1 << 22) if name == "irreg" else 1 << 16)
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
        balls = np.stack([np.concatenate([p[rng.integers(0, len(p), 64), :3], rng.uniform(20, 80, (64, 1))], 1) for p in parts])
        balls_t = torch.from_numpy(balls.astype(np.float32)).to(dev)
        near = torch.empty((1024, 64, 8, 2), dtype=torch.float32, device=dev)
        cnt = torch.empty((1024, 64), dtype=torch.int32, device=dev)
        ms = timed(torch, lambda: ctx.query_scene_batch_spheres_into(balls_t.data_ptr(), 64, batch, 8, near.data_ptr(),
                                                                     cnt.data_ptr()), args.steps, args.warmup)
        stale = sum(int(R.host_lbvh(p)["stale_nodes"] > 0) for p in parts)

        def per_scene():
            off = 0
            for b, p in enumerate(parts):
                brute(torch, recs[off:off + len(p)], balls_t[b], 8)
                off += len(p)
        bms = timed(torch, per_scene, max(1, args.steps // 2), 1)
        row = {"scenes": 1024, "spheres": int(sum(counts)), "balls_per_scene": 64, "k": 8, "members_with_stale_boxes": stale,
               "ms": ms, "brute_ms_per_scene_loop": bms, "speedup_vs_brute": round(bms / ms, 1),
               "mean_count": round(float(cnt.double().mean()), 3)}
        result["workloads"][key] = row
        print(key, row, file=sys.stderr, flush=True)
        batch.free()
    # 4. refit: kernel times of the complete-box refit against the query kernel
    if want("refit"):
        from torch.profiler import ProfilerActivity, profile
        rg, _ = R.host_scene("rgbbox")
        groups = np.zeros((1 << 20, 7), np.float32)
        groups[:, :3] = rng.uniform(0, 1024, ((1 << 20), 3))
        groups[:, 6] = rng.uniform(0.5, 3, 1 << 20)
        for g in range(6):   # coincident groups, whose boxes the fixed-sweep refit leaves stale
            groups[g * 40:(g + 1) * 40, :3] = (64 + 40 * g, 512, 512)
            groups[g * 40:(g + 1) * 40, 6] = 16
        for name, s in (("rgbbox", rg), ("groups2p20", groups)):
            s_t = torch.from_numpy(s).to(dev)
            pr = ctx.prepare_scene_device(64, 64, s_t, np.float32([0, 0, 1, 0, 0, 0, 40]))
            n = 1 << 16
            idx = rng.integers(0, len(s), n)
            balls = torch.from_numpy(np.ascontiguousarray(s[idx][:, [0, 1, 2, 6]])).to(dev)
            near = torch.empty((n, 8, 2), dtype=torch.float32, device=dev)
            cnt = torch.empty((n,), dtype=torch.int32, device=dev)

            def call():
                ctx.query_spheres_into(balls.data_ptr(), n, pr, 8, near.data_ptr(), cnt.data_ptr())
            ms = timed(torch, call, args.steps, args.warmup)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    call()
                torch.cuda.synchronize()
            us = {}
            for ev in prof.key_averages():
                for tag in ("prox_parents_kernel", "prox_refit_kernel", "prox_query_kernel"):
                    if tag in ev.key:
                        us[tag] = us.get(tag, 0.0) + ev.device_time_total / args.steps
            row = {"spheres": len(s), "balls": n, "k": 8, "stale_nodes": pr.info()["stale_nodes"], "call_ms": ms,
                   "refit_kernels_us": round(us.get("prox_parents_kernel", 0.0) + us.get("prox_refit_kernel", 0.0), 2),
                   "query_kernel_us": round(us.get("prox_query_kernel", 0.0), 2)}
            result["workloads"][f"refit_{name}"] = row
            print(f"refit_{name}", row, file=sys.stderr, flush=True)
            pr.free()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
