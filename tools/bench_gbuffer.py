#!/usr/bin/env python
"""The first-hit buffers of a frame (include/ray_b200.h ray_b200_render_gbuffer) against a colour frame of the same size
and sample count, and against building them from materialised camera rays; prints one JSON line.

    python tools/bench_gbuffer.py [--reps N] [--only WORKLOAD,...] [--out PATH]

For every workload, `gbuffer_ms` is the device time of one render_gbuffer_into call writing all five buffers and
`render_ms` that of render_into at the same size and spp (the context's CUDA events, ray_b200_context_last_render_ms; the
median of --reps runs, default 5, alternated, after one untimed run of each that loads the kernels and records the
colour frame's learned claim order).  `ratio` = gbuffer_ms / render_ms.  Workloads with "route" also time what a caller
does without the call: camera rays made on the host (raytracers_b200.camera_rays) and copied to the device, trace_hits and
trace_paths(max_depth = 1) over them, and the per-pixel reduction in torch (`route_ms`, host clock around all of it,
ending in a synchronisation; `route_queries_ms`, the two queries' device times alone).

Every timed output is checked in the same run against the rule, evaluated in torch on the GPU's own trace_hits /
trace_paths over the camera rays of the whole frame: `differing_values` counts the values of the five buffers that
differ, bit for bit and NaN-aware (the contract says 0).  The card's name and power limit are read in the same run.

- rgbbox / irreg at 1000x1000 and 1, 16, 64 spp (16 spp with the materialised-ray route);
- rgbbox / irreg at 256x256 and 64 spp: a small frame at many samples, where a colour frame spreads its samples over a
  warp's slots and the G-buffer, which never does, keeps each pixel's samples in one slot;
- random1M at 2000x2000 and 16 spp: the 1 M-sphere scene (seed 1).
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

WORKLOADS = [("rgbbox_1000_1spp", "rgbbox", 1000, 1, False), ("rgbbox_1000_16spp", "rgbbox", 1000, 16, True),
             ("rgbbox_1000_64spp", "rgbbox", 1000, 64, False), ("irreg_1000_1spp", "irreg", 1000, 1, False),
             ("irreg_1000_16spp", "irreg", 1000, 16, True), ("irreg_1000_64spp", "irreg", 1000, 64, False),
             ("rgbbox_256_64spp", "rgbbox", 256, 64, False), ("irreg_256_64spp", "irreg", 256, 64, False),
             ("random1M_2000_16spp", "random", 2000, 16, False)]
OUTPUTS = ("id", "depth", "normal", "albedo", "coverage")


def rule(torch, hits, sky, colours, spp):
    """The buffers of ray_b200_render_gbuffer from hit records [n, spp, 8] and sky colours [n, spp, 3] (trace_hits and
    trace_paths(max_depth = 1) of the camera rays), in torch on the device: in-order f32 sums, then 1/spp."""
    sphere = hits[..., 1].contiguous().view(torch.int32)
    hit = sphere >= 0
    albedo = torch.where(hit[..., None], colours[sphere.clamp(min=0).long()], sky)
    normal = hits[..., 5:8]
    n_sum, a_sum = normal[:, 0].clone(), albedo[:, 0].clone()
    for s in range(1, spp):
        n_sum = n_sum + normal[:, s]
        a_sum = a_sum + albedo[:, s]
    if spp > 1:
        inv = torch.tensor(1.0, dtype=torch.float32, device=hits.device) / torch.tensor(float(spp), dtype=torch.float32,
                                                                                      device=hits.device)
        n_sum, a_sum = inv * n_sum, inv * a_sum
    return {"id": sphere[:, 0], "depth": hits[:, 0, 0], "normal": n_sum, "albedo": a_sum,
            "coverage": hit.sum(1, dtype=torch.int32)}


def differing(torch, got, want):
    bad = 0
    for k in OUTPUTS:
        a, b = got[k].reshape(-1), want[k].reshape(-1)
        if a.dtype == torch.float32:
            na, nb = torch.isnan(a), torch.isnan(b)
            bad += int(((na != nb) | (~na & (a.view(torch.int32) != b.view(torch.int32)))).sum())
        else:
            bad += int((a != b).sum())
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    ctx = R.Context(device=0)
    records = {}
    med = lambda xs: round(statistics.median(xs), 3)   # noqa: E731
    for key, name, size, spp, route in WORKLOADS:
        if only and key not in only:
            continue
        spheres, cam = R.host_scene(name, 1 << 20, 1) if name == "random" else R.host_scene(name)
        scene = ctx.scene_from_arrays(spheres, cam)
        prepared = ctx.prepare_scene(size, size, scene)
        colours = torch.from_numpy(spheres[:, 3:6].copy()).cuda()
        h = w = size
        shapes = {"id": ((h, w), torch.int32), "depth": ((h, w), torch.float32), "normal": ((h, w, 3), torch.float32),
                  "albedo": ((h, w, 3), torch.float32), "coverage": ((h, w), torch.int32)}
        bufs = {k: torch.empty(s, dtype=t, device="cuda") for k, (s, t) in shapes.items()}
        pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

        def gbuffer():
            ctx.render_gbuffer_into(prepared, h, w, spp, *(bufs[k].data_ptr() for k in OUTPUTS))
            return ctx.last_render_ms()

        def render():
            ctx.render_into(pix.data_ptr(), h, w, prepared, spp=spp)
            return ctx.last_render_ms()

        def materialised():
            t0 = time.perf_counter()
            rays = torch.from_numpy(R.camera_rays(prepared.info()["camera"], h, w, spp).reshape(-1, 6)).cuda()
            hits = ctx.trace_hits(prepared, rays)
            q_ms = ctx.last_render_ms()
            sky = ctx.trace_paths(prepared, rays, max_depth=1)[0]
            q_ms += ctx.last_render_ms()
            buf = torch.cat([hits["t"][:, None], hits["sphere"].view(torch.float32)[:, None], hits["p"], hits["normal"]], 1)
            out = rule(torch, buf.view(-1, spp, 8), sky.view(-1, spp, 3), colours, spp)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), q_ms, out

        gbuffer(), render()
        t_g, t_r, t_route, t_q = [], [], [], []
        for _ in range(args.reps):
            t_g.append(gbuffer())
            t_r.append(render())
            if route:
                ms, q_ms, out = materialised()
                t_route.append(ms)
                t_q.append(q_ms)
                del out
        ctx.sync()
        # the check: the rule on the GPU's own queries over every camera ray of the frame (the route's own output)
        _, _, want = materialised()
        bad = differing(torch, bufs, want)
        del want
        torch.cuda.empty_cache()
        rec = {"scene": name, "size": size, "spp": spp, "gbuffer_ms": med(t_g), "render_ms": med(t_r),
               "ratio": round(med(t_g) / med(t_r), 3), "covered_pixels": int((bufs["coverage"] > 0).sum()),
               "differing_values": bad}
        if route:
            rec.update({"route_ms": med(t_route), "route_queries_ms": med(t_q),
                        "speedup_vs_route": round(med(t_route) / med(t_g), 2)})
        records[key] = rec
        print(key, rec, file=sys.stderr, flush=True)
        prepared.free(); scene.free()
        del bufs, pix
        torch.cuda.empty_cache()
    ctx.close()
    line = json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                       "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "reps": args.reps, "workloads": records})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if all(r["differing_values"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
