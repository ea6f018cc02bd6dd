#!/usr/bin/env python
"""Several views in one launch (include/ray_b200.h ray_b200_render_views_into) against one launch per view; prints one
JSON line.

    python tools/bench_views.py [--reps N] [--only WORKLOAD,...]

For every workload, V views of one scene through one render_views_into call (`views_ms`) against the same V frames as
V render_into calls on V prepared scenes, one per camera (`per_view_ms`, the sum of the calls' device times), and as one
render_batch of the same V jobs (`batch_ms`, up to two frames in flight).  Device times are the context's CUDA events
(ray_b200_context_last_render_ms); each number is the median of --reps runs (default 3), the three forms alternated,
after one untimed run of each that loads the kernels and records the per-view scenes' learned claim order.
`prepare_ms` is the host time of preparing the V per-view scenes (scene_from_arrays + prepare_scene + a synchronisation),
which a caller without views pays on top of per_view_ms; the views call uses one scene prepared once.
`differing_pixels` counts the pixels of the views call that differ from the per-view renders and from the batch (the
contract says 0).  The card's name and power limit are read in the same run.

- orbit64_irreg_256_16spp: 64 cameras on an orbit around irreg's look_at, 256x256, 16 spp;
- cube6_rgbbox_512_64spp: 6 cube-map faces (fov 90) from rgbbox's camera position, 512x512, 64 spp (the up and down faces
  lean 0.001 off vertical: a camera looking along vup has no image, ray.fut:93-107);
- random1M_8views_500_4spp: 8 cameras around the 1 M-sphere scene (seed 1), 500x500, 4 spp;
- moved1_irreg_1000_1spp: irreg from one moved camera, 1000x1000, 1 spp (n_views = 1: another camera without preparing
  the scene again).
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def orbit(cam7, n, radius_scale=1.0, height=0.3):
    """n cameras evenly around cam7's look_at, at cam7's distance times radius_scale, `height` radians up."""
    c = np.asarray(cam7, np.float64)
    at = c[3:6]
    r = float(np.linalg.norm(c[0:3] - at)) * radius_scale
    out = []
    for k in range(n):
        a = 2 * math.pi * k / n
        lf = at + r * np.array([math.cos(height) * math.sin(a), math.sin(height), math.cos(height) * math.cos(a)])
        out.append(np.concatenate([lf, at, [c[6]]]))
    return np.asarray(out, np.float32)


def cube(cam7):
    eye = np.asarray(cam7, np.float64)[0:3]
    dirs = [(1, 0, 0), (-1, 0, 0), (0.001, 1, 0), (0.001, -1, 0), (0, 0, 1), (0, 0, -1)]
    return np.asarray([np.concatenate([eye, eye + np.array(d), [90.0]]) for d in dirs], np.float32)


def moved(cam7):
    c = np.array(cam7, np.float32)
    c[0:3] = c[0:3] + np.float32([8.0, 3.0, -4.0])
    return c[None]


WORKLOADS = [("orbit64_irreg_256_16spp", "irreg", 256, 16, lambda c: orbit(c, 64)),
             ("cube6_rgbbox_512_64spp", "rgbbox", 512, 64, cube),
             ("random1M_8views_500_4spp", "random", 500, 4, lambda c: orbit(c, 8, 0.8)),
             ("moved1_irreg_1000_1spp", "irreg", 1000, 1, moved)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    ctx = R.Context(device=0)
    records = {}
    for key, name, size, spp, make_cams in WORKLOADS:
        if only and key not in only:
            continue
        spheres, cam = R.host_scene(name, 1 << 20, 1) if name == "random" else R.host_scene(name)
        cams = make_cams(cam)
        V = len(cams)
        scene = ctx.scene_from_arrays(spheres, cam)
        prepared = ctx.prepare_scene(size, size, scene)
        got = torch.empty((V, size, size), dtype=torch.int32, device="cuda")
        each = torch.empty((V, size, size), dtype=torch.int32, device="cuda")
        batch = torch.empty((V, size, size), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

        def prepare_all():
            t0 = time.perf_counter()
            out = []
            for c in cams:
                sc = ctx.scene_from_arrays(spheres, c)
                out.append((sc, ctx.prepare_scene(size, size, sc)))
            ctx.sync()
            return out, 1e3 * (time.perf_counter() - t0)

        per_view, prep_ms = prepare_all()
        jobs = [dict(prepared=pr, h=size, w=size, spp=spp, out_dev=batch[v].data_ptr()) for v, (_, pr) in enumerate(per_view)]

        def views():
            ctx.render_views_into(prepared, cams, size, size, spp, got.data_ptr())
            return ctx.last_render_ms()

        def one_by_one():
            ms = 0.0
            for v, (_, pr) in enumerate(per_view):
                ctx.render_into(each[v].data_ptr(), size, size, pr, spp=spp)
                ms += ctx.last_render_ms()
            return ms

        def batched():
            ctx.render_batch(jobs)
            return ctx.last_render_ms()

        views(), one_by_one(), batched()   # load the kernels, record the per-view scenes' learned claim order
        t_views, t_each, t_batch, t_prep = [], [], [], [prep_ms]
        for rep in range(args.reps):
            t_views.append(views())
            t_each.append(one_by_one())
            t_batch.append(batched())
            if rep:   # preparing the per-view scenes again, for the spread of prepare_ms
                for sc, pr in per_view:
                    pr.free(); sc.free()
                per_view, ms = prepare_all()
                t_prep.append(ms)
                jobs = [dict(prepared=pr, h=size, w=size, spp=spp, out_dev=batch[v].data_ptr()) for v, (_, pr) in enumerate(per_view)]
        ctx.sync()
        med = lambda xs: round(statistics.median(xs), 3)   # noqa: E731
        records[key] = {"scene": name, "views": V, "size": size, "spp": spp,
                        "views_ms": med(t_views), "per_view_ms": med(t_each), "batch_ms": med(t_batch),
                        "prepare_ms": med(t_prep), "per_view_with_prepare_ms": round(med(t_each) + med(t_prep), 3),
                        "speedup_vs_per_view": round(med(t_each) / med(t_views), 3),
                        "speedup_vs_batch": round(med(t_batch) / med(t_views), 3),
                        "differing_pixels": int((got != each).sum()) + int((got != batch).sum())}
        print(key, records[key], file=sys.stderr, flush=True)
        for sc, pr in per_view:
            pr.free(); sc.free()
        prepared.free(); scene.free()
        del got, each, batch
    ctx.close()
    print(json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                      "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "reps": args.reps, "workloads": records}))
    return 0 if all(r["differing_pixels"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
