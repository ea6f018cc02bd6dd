#!/usr/bin/env python
"""An animation loop over a scene whose spheres live in a CUDA tensor: each frame a torch op moves every sphere centre,
then the frame is rendered, by two routes; prints one JSON line.

    python tools/bench_dynamic.py [--frames N] [--only WORKLOAD,...] [--out PATH]

  (a) device route: PreparedScene.update(spheres) (ray_b200_prepared_update: the LBVH rebuilt from the tensor in place,
      no host copy), then render_into;
  (b) host route: spheres.cpu(), scene_from_arrays, prepare_scene (page-locked copy, H2D, device build), render_into,
      and freeing the prepared scene and the scene.

Per workload, medians over --frames timed frames (default 10, after 2 untimed ones), the routes alternating frame by
frame: `update_ms` is the host clock around update (the call blocks until its build's read-back), `build_ms` the
device time of the update's work (CUDA events around it on the context's stream, which is torch's current stream
here), `render_ms_a` / `render_ms_b` the render's device time (ray_b200_context_last_render_ms), and `loop_ms_a` /
`loop_ms_b` the host clock around one whole frame (move, rebuild, render, synchronise).  `update_share` =
update_ms / loop_ms_a.  `differing_pixels` counts the pixels of every frame where the two routes differ (the contract
says 0).  The card's name and power limit are read in the same run.

- irreg at 1000x1000, 1 and 16 spp;
- a 2^16-sphere random scene (seed 1) at 1000x1000, 1 and 16 spp;
- the 1 M-sphere random scene (seed 1) at 2000x2000, 1 and 16 spp.
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

WORKLOADS = [("irreg_1000_1spp", "irreg", 0, 1000, 1), ("irreg_1000_16spp", "irreg", 0, 1000, 16),
             ("random64k_1000_1spp", "random", 1 << 16, 1000, 1), ("random64k_1000_16spp", "random", 1 << 16, 1000, 16),
             ("random1M_2000_1spp", "random", 1 << 20, 2000, 1), ("random1M_2000_16spp", "random", 1 << 20, 2000, 16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    ctx = R.Context(device=0)
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)     # the build's events and the torch ops share one stream
    records = {}
    med = lambda xs: round(statistics.median(xs), 3)   # noqa: E731
    for key, name, n, size, spp in WORKLOADS:
        if only and key not in only:
            continue
        spheres, cam = R.host_scene(name, n, 1) if name == "random" else R.host_scene(name)
        base = torch.from_numpy(spheres).cuda()
        extent = float((base[:, :3].max(0).values - base[:, :3].min(0).values).max())
        step = torch.tensor([1.0, 0.5, -0.75, 0, 0, 0, 0], device="cuda") * (extent / 400)
        cur = base.clone()
        h = w = size
        pix_a = torch.empty((h, w), dtype=torch.int32, device="cuda")
        pix_b = torch.empty((h, w), dtype=torch.int32, device="cuda")
        prepared = ctx.prepare_scene_device(h, w, cur, cam)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = {k: [] for k in ("update", "build", "render_a", "render_b", "loop_a", "loop_b")}
        bad = 0
        for frame in range(2 + args.frames):
            timed = frame >= 2
            torch.cuda.synchronize()
            # (a) move on the GPU, rebuild in place, render
            t0 = time.perf_counter()
            torch.add(base, step * (frame + 1), out=cur)
            t1 = time.perf_counter()
            ev0.record(stream)
            prepared.update(cur)
            ev1.record(stream)
            t2 = time.perf_counter()
            ctx.render_into(pix_a.data_ptr(), h, w, prepared, spp=spp)
            ms_a = ctx.last_render_ms()
            ctx.sync()
            t3 = time.perf_counter()
            # (b) the same records through the host
            torch.add(base, step * (frame + 1), out=cur)
            host = cur.cpu()
            sc = ctx.scene_from_arrays(host.numpy(), cam)
            pr_b = ctx.prepare_scene(h, w, sc)
            ctx.render_into(pix_b.data_ptr(), h, w, pr_b, spp=spp)
            ms_b = ctx.last_render_ms()
            ctx.sync()
            pr_b.free(); sc.free()
            t4 = time.perf_counter()
            bad += int((pix_a != pix_b).sum())
            if timed:
                t["update"].append(1e3 * (t2 - t1))
                t["build"].append(ev0.elapsed_time(ev1))
                t["render_a"].append(ms_a)
                t["render_b"].append(ms_b)
                t["loop_a"].append(1e3 * (t3 - t0))
                t["loop_b"].append(1e3 * (t4 - t3))
        rec = {"scene": name, "spheres": len(spheres), "size": size, "spp": spp, "frames": args.frames,
               "update_ms": med(t["update"]), "build_ms": med(t["build"]), "render_ms_a": med(t["render_a"]),
               "render_ms_b": med(t["render_b"]), "loop_ms_a": med(t["loop_a"]), "loop_ms_b": med(t["loop_b"]),
               "update_share": round(med(t["update"]) / med(t["loop_a"]), 3),
               "speedup": round(med(t["loop_b"]) / med(t["loop_a"]), 2), "upload_bytes_a": prepared.upload_bytes(),
               "differing_pixels": bad}
        records[key] = rec
        print(key, rec, file=sys.stderr, flush=True)
        prepared.free()
        del base, cur, pix_a, pix_b
        torch.cuda.empty_cache()
    ctx.set_stream(None)
    ctx.close()
    line = json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                       "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "frames": args.frames, "workloads": records})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if all(r["differing_pixels"] == 0 and r["upload_bytes_a"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
