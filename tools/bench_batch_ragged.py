#!/usr/bin/env python
"""Many small scenes of different sizes animated on the GPU: each step a torch op moves every sphere centre of an
[N, 7] tensor, then every scene is rebuilt and one frame of each is rendered (or a fan of rays traced in each), by two
routes that give the same answers; prints one JSON line.

    python tools/bench_batch_ragged.py [--steps N] [--warmup W] [--only WORKLOAD,...] [--out PATH]

  (ragged)       SceneBatch.update(counts=...) (one build of all B trees, one read-back), then one render_scene_batch_into
                 launch (or one trace_scene_batch_hits_into launch);
  (render_batch) B x PreparedScene.update, then one ray_b200_render_batch of the B frames (or B x trace_hits_into).

Per workload, medians over --steps timed steps (default 5, after --warmup untimed ones, default 2), the routes
alternating step by step: `step_ms_*` is the host clock around one whole step (move, rebuild, render or trace,
synchronise), `update_ms_*` the host clock around the rebuild, `work_ms_*` the device time of the renders or queries
(CUDA events on the context's stream, torch's current stream here).  `differing_values` counts the pixels or hit-record
words of every timed step where the per-scene route differs from the batch (the contract says 0).  The card's name and
power limit are read in the same run.

- 1024 random scenes of 16 to 256 spheres (seeded draw) at 84 x 84, 1 spp;
- one random scene of 2^20 spheres next to 1023 of 64, at 84 x 84, 1 spp (one large member among many small ones);
- the first workload's scenes, a fan of 1024 rays per scene (from a point outside the scene towards its spheres) to
  their closest hits.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("b1024_n16to256_84_1spp", "render"), ("b1024_skewed_2p20_84_1spp", "render"), ("b1024_n16to256_hits_1024", "hits")]
ROUTES = ("ragged", "render_batch")


def counts_of(key):
    import numpy as np
    if "skewed" in key:
        return np.array([1 << 20] + [64] * 1023, np.int64)
    return np.random.default_rng(7).integers(16, 257, 1024).astype(np.int64)


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
    ctx = R.Context(device=0)
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)
    records = {}
    med = lambda xs: round(statistics.median(xs), 3)   # noqa: E731
    h = w = 84
    m = 1024
    for key, work in WORKLOADS:
        if only and key not in only:
            continue
        counts = counts_of(key)
        B = len(counts)
        off = np.concatenate([[0], np.cumsum(counts)])
        parts = [R.host_scene("random", int(n), 1 + b) for b, n in enumerate(counts)]
        base = torch.from_numpy(np.ascontiguousarray(np.concatenate([s for s, _ in parts]), np.float32)).cuda()
        cams = np.stack([c for _, c in parts])
        extent = float((base[:counts[0], :3].max(0).values - base[:counts[0], :3].min(0).values).max())
        move = torch.tensor([1.0, 0.5, -0.75, 0, 0, 0, 0], device="cuda") * (extent / 400)
        cur = base.clone()
        batch = ctx.prepare_scene_batch(h, w, cur, cams, counts=counts)
        scenes = [ctx.prepare_scene_device(h, w, cur[off[b]:off[b + 1]], cams[b]) for b in range(B)]
        if work == "render":
            out = {r: torch.empty((B, h, w), dtype=torch.int32, device="cuda") for r in ROUTES}
            jobs = [dict(prepared=scenes[b], h=h, w=w, spp=1, out_dev=out["render_batch"][b].data_ptr()) for b in range(B)]
        else:
            rng = np.random.default_rng(3)
            rays = np.empty((B, m, 6), np.float32)
            for b, (s, _) in enumerate(parts):   # a fan from a point beside the scene towards its spheres
                lo, hi = s[:, :3].min(0), s[:, :3].max(0)
                rays[b, :, :3] = hi + (hi - lo) * 0.5
                rays[b, :, 3:] = s[rng.integers(0, len(s), m), :3] - rays[b, :, :3]
            rays = torch.from_numpy(rays).cuda()
            out = {r: torch.empty((B, m, 8), dtype=torch.float32, device="cuda") for r in ROUTES}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = {f"{k}_{r}": [] for k in ("step", "update", "work") for r in ROUTES}
        bad = 0
        for step in range(args.warmup + args.steps):
            timed = step >= args.warmup
            for r in ROUTES:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                torch.add(base, move * (step + 1), out=cur)
                t1 = time.perf_counter()
                if r == "ragged":
                    batch.update(cur, counts=counts)
                else:
                    for b in range(B):
                        scenes[b].update(cur[off[b]:off[b + 1]])
                t2 = time.perf_counter()
                ev0.record(stream)
                if work == "render" and r == "ragged":
                    ctx.render_scene_batch_into(batch, h, w, 1, out[r].data_ptr())
                elif work == "render":
                    ctx.render_batch(jobs)
                elif r == "ragged":
                    ctx.trace_scene_batch_hits_into(rays.data_ptr(), m, batch, out[r].data_ptr())
                else:
                    for b in range(B):
                        ctx.trace_hits_into(rays[b].data_ptr(), m, scenes[b], out[r][b].data_ptr())
                ev1.record(stream)
                ctx.sync()
                t3 = time.perf_counter()
                if timed:
                    t[f"step_{r}"].append(1e3 * (t3 - t0))
                    t[f"update_{r}"].append(1e3 * (t2 - t1))
                    t[f"work_{r}"].append(ev0.elapsed_time(ev1))
            if timed:
                bad += int((out["render_batch"].view(torch.int32) != out["ragged"].view(torch.int32)).sum())
        rec = {"work": work, "scenes": B, "spheres": int(off[-1]), "min_count": int(counts.min()), "max_count": int(counts.max()),
               "size": h, "spp": 1, "rays_per_scene": m if work == "hits" else 0, "steps": args.steps}
        rec.update({f"{k}_ms_{r}": med(t[f"{k}_{r}"]) for k in ("step", "update", "work") for r in ROUTES})
        rec["step_speedup"] = round(med(t["step_render_batch"]) / med(t["step_ragged"]), 2)
        rec["update_speedup"] = round(med(t["update_render_batch"]) / med(t["update_ragged"]), 2)
        rec["work_speedup"] = round(med(t["work_render_batch"]) / med(t["work_ragged"]), 3)
        rec["differing_values"] = bad
        records[key] = rec
        print(key, rec, file=sys.stderr, flush=True)
        batch.free()
        for p in scenes:
            p.free()
        del base, cur, out
        torch.cuda.empty_cache()
    ctx.set_stream(None)
    ctx.close()
    line = json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                       "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "steps": args.steps,
                       "warmup": args.warmup, "workloads": records})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if all(r["differing_values"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
