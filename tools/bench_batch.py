#!/usr/bin/env python
"""Many small scenes animated on the GPU: each step a torch op moves every sphere centre of a [B, n, 7] tensor, then
every scene is rebuilt and one frame of each is rendered, by three routes; prints one JSON line.

    python tools/bench_batch.py [--steps N] [--warmup W] [--only WORKLOAD,...] [--out PATH]

  (batch)        SceneBatch.update (one build of all B trees, one read-back), then one render_scene_batch_into launch;
  (render_batch) B x PreparedScene.update, then one ray_b200_render_batch of the B frames (two in flight);
  (render_into)  B x PreparedScene.update, then B x render_into.

Per workload, medians over --steps timed steps (default 5, after --warmup untimed ones, default 2), the routes
alternating step by step: `step_ms_*` is the host clock around one whole step (move, rebuild, render, synchronise),
`update_ms_*` the host clock around the rebuild (every update call blocks on its build's read-back), `render_ms_*` the
device time of the renders (CUDA events around them on the context's stream, which is torch's current stream here).
`differing_pixels` counts the pixels of every timed step's frames where a per-scene route differs from the batch (the
contract says 0).  The card's name and power limit are read in the same run.

- B = 1024 scenes of 64 random spheres at 84 x 84, 1 spp;
- B = 256 scenes of 1024 random spheres at 128 x 128, 4 spp;
- B = 16 scenes of 10 000 random spheres at 256 x 256, 16 spp;
- B = 1: irreg at 1000 x 1000, 1 spp (the batch route against render_into of one prepared scene: the cost of the kind's
  per-segment root-box table read).
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

WORKLOADS = [("b1024_n64_84_1spp", "random", 1024, 64, 84, 1), ("b256_n1024_128_4spp", "random", 256, 1024, 128, 4),
             ("b16_n10000_256_16spp", "random", 16, 10000, 256, 16), ("b1_irreg_1000_1spp", "irreg", 1, 0, 1000, 1)]
ROUTES = ("batch", "render_batch", "render_into")


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
    ctx.set_stream(stream.cuda_stream)     # the events and the torch ops share the context's stream
    records = {}
    med = lambda xs: round(statistics.median(xs), 3)   # noqa: E731
    for key, name, B, n, size, spp in WORKLOADS:
        if only and key not in only:
            continue
        recs, cams = [], []
        for b in range(B):
            s, c = R.host_scene(name, n, 1 + b) if name == "random" else R.host_scene(name)
            recs.append(s)
            cams.append(c)
        base = torch.from_numpy(np.ascontiguousarray(np.stack(recs), np.float32)).cuda()
        cams = np.stack(cams)
        B, n = base.shape[0], base.shape[1]
        extent = float((base[0, :, :3].max(0).values - base[0, :, :3].min(0).values).max())
        move = torch.tensor([1.0, 0.5, -0.75, 0, 0, 0, 0], device="cuda") * (extent / 400)
        cur = base.clone()
        h = w = size
        batch = ctx.prepare_scene_batch(h, w, cur, cams)
        scenes = [ctx.prepare_scene_device(h, w, cur[b], cams[b]) for b in range(B)]
        pix = {r: torch.empty((B, h, w), dtype=torch.int32, device="cuda") for r in ROUTES}
        jobs = [dict(prepared=scenes[b], h=h, w=w, spp=spp, out_dev=pix["render_batch"][b].data_ptr()) for b in range(B)]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = {f"{k}_{r}": [] for k in ("step", "update", "render") for r in ROUTES}
        bad = {r: 0 for r in ROUTES[1:]}
        for step in range(args.warmup + args.steps):
            timed = step >= args.warmup
            for r in ROUTES:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                torch.add(base, move * (step + 1), out=cur)
                t1 = time.perf_counter()
                if r == "batch":
                    batch.update(cur)
                else:
                    for b in range(B):
                        scenes[b].update(cur[b])
                t2 = time.perf_counter()
                ev0.record(stream)
                if r == "batch":
                    ctx.render_scene_batch_into(batch, h, w, spp, pix[r].data_ptr())
                elif r == "render_batch":
                    ctx.render_batch(jobs)
                else:
                    for b in range(B):
                        ctx.render_into(pix[r][b].data_ptr(), h, w, scenes[b], spp=spp)
                ev1.record(stream)
                ctx.sync()
                t3 = time.perf_counter()
                if timed:
                    t[f"step_{r}"].append(1e3 * (t3 - t0))
                    t[f"update_{r}"].append(1e3 * (t2 - t1))
                    t[f"render_{r}"].append(ev0.elapsed_time(ev1))
            if timed:
                for r in ROUTES[1:]:
                    bad[r] += int((pix[r] != pix["batch"]).sum())
        rec = {"scene": name, "scenes": B, "spheres": n, "size": size, "spp": spp, "steps": args.steps}
        rec.update({f"{k}_ms_{r}": med(t[f"{k}_{r}"]) for k in ("step", "update", "render") for r in ROUTES})
        rec.update({f"step_speedup_vs_{r}": round(med(t[f"step_{r}"]) / med(t["step_batch"]), 2) for r in ROUTES[1:]})
        rec.update({f"render_speedup_vs_{r}": round(med(t[f"render_{r}"]) / med(t["render_batch"]), 3) for r in ROUTES[1:]})
        rec["differing_pixels"] = sum(bad.values())
        records[key] = rec
        print(key, rec, file=sys.stderr, flush=True)
        batch.free()
        for p in scenes:
            p.free()
        del base, cur, pix
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
    return 0 if all(r["differing_pixels"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
