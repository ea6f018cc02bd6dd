#!/usr/bin/env python
"""Progressive rendering (include/ray_b200.h ray_b200_render_accumulate) against one-shot renders; prints one JSON line.

    python tools/bench_progressive.py [--reps N] [--only WORKLOAD,...]

For every workload, the frame of one render_into at the total spp (`oneshot_ms`) against the same frame accumulated in
chunks: `total_ms` = the sum of the chunks' device times, `longest_ms` = the longest single call, `wall_ms` = host time of
the whole chain (one synchronisation per call, as a preview loop has), and `calls`.  Device times are the context's CUDA
events (ray_b200_context_last_render_ms); each number is the median of --reps runs (default 3), one-shot renders and
chains alternated, after one untimed run of each that loads the kernels.  `differing_pixels` counts the pixels of the
last chain's frame that differ from the one-shot frame (the contract says 0).  The card's name and power limit are read
in the same run.

- scenes_1000_64spp_chunk{64,16,4,1}: rgbbox and irreg at 1000x1000, 64 spp (bench.py's frames), in chunks of 64, 16, 4
  and 1 samples (times are the two scenes' sums);
- irreg_4000_256spp_chunk16: irreg at 4000x4000, 256 spp, 16 chunks of 16;
- random1M_2000_16spp_chunk4: the 1 M-sphere scene (seed 1) at 2000x2000, 16 spp, chunks of 4.
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

WORKLOADS = [("scenes_1000_64spp_chunk64", ("rgbbox", "irreg"), 1000, 64, 64),
             ("scenes_1000_64spp_chunk16", ("rgbbox", "irreg"), 1000, 64, 16),
             ("scenes_1000_64spp_chunk4", ("rgbbox", "irreg"), 1000, 64, 4),
             ("scenes_1000_64spp_chunk1", ("rgbbox", "irreg"), 1000, 64, 1),
             ("irreg_4000_256spp_chunk16", ("irreg",), 4000, 256, 16),
             ("random1M_2000_16spp_chunk4", ("random",), 2000, 16, 4)]


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
    prepared = {}

    def scene(name, size):
        if (name, size) not in prepared:
            sc = ctx.scene_random(1 << 20, 1) if name == "random" else ctx.scene(name)
            prepared[(name, size)] = ctx.prepare_scene(size, size, sc)
        return prepared[(name, size)]

    records = {}
    for key, names, size, spp, chunk in WORKLOADS:
        if only and key not in only:
            continue
        want = {n: torch.empty((size, size), dtype=torch.int32, device="cuda") for n in names}
        got = {n: torch.empty((size, size), dtype=torch.int32, device="cuda") for n in names}
        accum = torch.empty((size, size, 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        splits = [(s, min(s + chunk, spp)) for s in range(0, spp, chunk)]

        def oneshot():
            ms = 0.0
            for n in names:
                ctx.render_into(want[n].data_ptr(), size, size, scene(n, size), spp=spp)
                ms += ctx.last_render_ms()
            return ms

        def chain():
            calls = []
            t0 = time.perf_counter()
            for n in names:
                for a, b in splits:
                    ctx.render_accumulate_into(accum.data_ptr(), size, size, scene(n, size), a, b, got[n].data_ptr())
                    calls.append(ctx.last_render_ms())   # (synchronises: the preview loop's read-back point)
            return sum(calls), max(calls), 1e3 * (time.perf_counter() - t0), len(calls)

        oneshot(), chain()   # load the kernels, record the learned claim order
        one, chained = [], []
        for _ in range(args.reps):
            one.append(oneshot())
            chained.append(chain())
        ctx.sync()
        diff = sum(int((got[n] != want[n]).sum()) for n in names)
        med = lambda i: round(statistics.median(c[i] for c in chained), 3)   # noqa: E731
        records[key] = {"scenes": list(names), "size": size, "spp": spp, "chunk": chunk, "calls": chained[0][3],
                        "oneshot_ms": round(statistics.median(one), 3), "total_ms": med(0), "longest_ms": med(1),
                        "wall_ms": med(2), "differing_pixels": diff}
        print(key, records[key], file=sys.stderr, flush=True)
        del want, got, accum
    ctx.close()
    print(json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                      "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "reps": args.reps, "workloads": records}))
    return 0 if all(r["differing_pixels"] == 0 for r in records.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
