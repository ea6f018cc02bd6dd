#!/usr/bin/env python
"""Ray queries on many scenes: one scene-batch query of m rays per scene against B single-scene queries on the members,
by two routes; prints one JSON line and writes it to --out.

    python tools/bench_batch_rays.py [--steps N] [--warmup W] [--only WORKLOAD,...] [--out PATH]

  (batch)   one ray_b200_scene_batch_trace_* call over the [B, m] rays;
  (members) B calls of the single-scene query (ray_b200_trace_*), one per member, on the same stream.

The members are made with SceneBatch.member before the timing starts (a device copy of each member's arrays, which the
per-scene route needs and a caller would keep), so neither route's time includes a build or a copy.  Per workload,
medians over --steps timed runs (default 7, after --warmup untimed ones, default 2), the routes alternating run by run:
`ms_*` is the device time of the route's calls (CUDA events around them on the context's stream).  `differing_records`
counts the output values of every timed run where the member route differs from the batch (the contract says 0).  The
card's name and power limit are read in the same run.

- B = 1024 scenes of 64 random spheres, a 1024-ray horizontal fan from each scene's centre (a lidar sweep), trace_hits;
- B = 256 scenes of 1024 random spheres, 4096 ranged shadow rays per scene (unit directions toward a light above the
  scene, t_max = the light's distance), trace_occluded;
- B = 16 scenes of 10 000 random spheres, 2^16 random rays per scene, trace_multi_hits with k = 4;
- B = 1: irreg, 2^22 random rays, trace_hits (the batch route against trace_hits of one prepared scene: the cost of the
  batch kind's per-segment division and root-box read).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# key, scene, B, n, rays per scene, query
WORKLOADS = [("b1024_n64_fan1024_hits", "random", 1024, 64, 1024, "hits"),
             ("b256_n1024_shadow4096_occluded", "random", 256, 1024, 4096, "occluded"),
             ("b16_n10000_random65536_multi4", "random", 16, 10000, 1 << 16, "multi_hits"),
             ("b1_irreg_random4194304_hits", "irreg", 1, 0, 1 << 22, "hits")]
ROUTES = ("batch", "members")
K = 4


def scene_box(s):
    return (s[:, :3] - s[:, 6:7]).min(0), (s[:, :3] + s[:, 6:7]).max(0)


def make_rays(np, kind, s, m, seed):
    """[m, 6] or, for shadow rays, [m, 8] float32 rays of one scene's records s"""
    lo, hi = scene_box(s)
    rng = np.random.default_rng(seed)
    if kind == "fan":
        a = np.linspace(0, 2 * np.pi, m, endpoint=False)
        o = np.broadcast_to((lo + hi) / 2, (m, 3))
        d = np.stack([np.cos(a), np.zeros(m), np.sin(a)], 1)
        return np.ascontiguousarray(np.concatenate([o, d], 1), np.float32)
    o = rng.uniform(lo, hi, (m, 3)).astype(np.float32)
    if kind == "shadow":
        light = np.float32([(lo[0] + hi[0]) / 2, hi[1] + (hi[1] - lo[1]), (lo[2] + hi[2]) / 2])
        v = light - o
        dist = np.sqrt((v * v).sum(1)).astype(np.float32)
        return np.ascontiguousarray(np.concatenate([o, np.full((m, 1), 1e-2), v / dist[:, None], dist[:, None] - 1e-4], 1),
                                    np.float32)
    d = rng.standard_normal((m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.ascontiguousarray(np.concatenate([o, d], 1), np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_batch_rays.json"))
    args = ap.parse_args()
    import numpy as np
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    ctx = R.Context(device=0)
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)     # the events share the context's stream
    records = {}
    med = lambda xs: round(statistics.median(xs), 4)   # noqa: E731
    for key, name, B, n, m, query in WORKLOADS:
        if only and key not in only:
            continue
        recs, cams = [], []
        for b in range(B):
            s, c = R.host_scene(name, n, 1 + b) if name == "random" else R.host_scene(name)
            recs.append(s)
            cams.append(c)
        spheres = np.ascontiguousarray(np.stack(recs), np.float32)
        B, n = spheres.shape[0], spheres.shape[1]
        ray_kind = "fan" if key.startswith("b1024") else "shadow" if query == "occluded" else "random"
        rays = torch.from_numpy(np.stack([make_rays(np, ray_kind, spheres[b], m, 100 + b) for b in range(B)])).cuda()
        ranged = rays.shape[2] == 8
        batch = ctx.prepare_scene_batch(16, 16, torch.from_numpy(spheres).cuda(), np.stack(cams))
        members = [batch.member(b) for b in range(B)]
        if query == "hits":
            out = {r: torch.empty((B, m, 8), dtype=torch.float32, device="cuda") for r in ROUTES}
        elif query == "occluded":
            out = {r: torch.empty((B, m), dtype=torch.uint8, device="cuda") for r in ROUTES}
        else:
            out = {r: torch.empty((B, m, K, 8), dtype=torch.float32, device="cuda") for r in ROUTES}
            counts = {r: torch.empty((B, m), dtype=torch.int32, device="cuda") for r in ROUTES}
        rp = rays.data_ptr()

        def batch_call():
            o = out["batch"].data_ptr()
            if query == "hits":
                ctx.trace_scene_batch_hits_into(rp, m, batch, o)
            elif query == "occluded":
                ctx.trace_scene_batch_occluded_ranged_into(rp, m, batch, o)
            else:
                ctx.trace_scene_batch_multi_hits_into(rp, m, batch, K, o, counts["batch"].data_ptr())

        def member_calls():
            for b in range(B):
                r, o = rays[b].data_ptr(), out["members"][b].data_ptr()
                if query == "hits":
                    ctx.trace_hits_into(r, m, members[b], o)
                elif query == "occluded":
                    ctx.trace_occluded_ranged_into(r, m, members[b], o)
                else:
                    ctx.trace_multi_hits_into(r, m, members[b], K, o, counts["members"][b].data_ptr())

        calls = {"batch": batch_call, "members": member_calls}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = {r: [] for r in ROUTES}
        bad = 0
        torch.cuda.synchronize()
        for step in range(args.warmup + args.steps):
            timed = step >= args.warmup
            for r in (ROUTES if step % 2 == 0 else ROUTES[::-1]):
                ev0.record(stream)
                calls[r]()
                ev1.record(stream)
                ctx.sync()
                if timed:
                    t[r].append(ev0.elapsed_time(ev1))
            if timed:
                a, b_ = out["batch"], out["members"]
                bad += int((a.view(torch.uint8) != b_.view(torch.uint8)).sum()) if query == "occluded" else \
                    int((a.view(torch.int32) != b_.view(torch.int32)).sum())
                if query == "multi_hits":
                    bad += int((counts["batch"] != counts["members"]).sum())
        rec = {"scene": name, "scenes": B, "spheres": n, "rays_per_scene": m, "query": query, "ranged": ranged,
               "k": K if query == "multi_hits" else None, "steps": args.steps, "members_prepared_outside_timing": True}
        rec.update({f"ms_{r}": med(t[r]) for r in ROUTES})
        rec.update({f"ms_min_{r}": round(min(t[r]), 4) for r in ROUTES})
        rec["speedup_vs_members"] = round(med(t["members"]) / med(t["batch"]), 3)
        rec["mrays_per_s_batch"] = round(B * m / med(t["batch"]) / 1e3, 1)
        rec["differing_records"] = bad
        records[key] = rec
        print(key, rec, file=sys.stderr, flush=True)
        for p in members:
            p.free()
        batch.free()
        del rays, out
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
    return 0 if all(r["differing_records"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
