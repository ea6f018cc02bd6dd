#!/usr/bin/env python
"""Adaptive progressive rendering (include/ray_b200.h ray_b200_render_adaptive) against whole-frame accumulation; prints
one JSON line.

    python tools/bench_adaptive.py [--reps N] [--only SCENE,...]

Scenes: irreg at 1000x1000 and the 1 M-sphere scene (seed 1) at 2000x2000.  Each is seeded with 4 samples everywhere
(render_accumulate(0, 4): the sums, counts of 4, and the 4-sample frame as the display buffer).  From that state every
workload times one call, after an untimed reset of the buffers:

- accumulate: render_accumulate(4, 8) of the whole frame, the baseline;
- adaptive n_add = 4 on the masks 100 %, 50 %, 10 % and 1 % random, 10 % as one block of whole 8x4 tiles, and 10 % with
  the largest change between the 4- and 8-sample means (the sum of the three channels' absolute differences, in torch: a
  caller's criterion), and a mask that selects nothing (the fixed cost of the selection pass and the launch);
- adaptive n_add = 1 (pixel-bound samples) on 10 % random.

Times are device times from the context's CUDA events (ray_b200_context_last_render_ms: the selection pass and the render
kernel), each the median of --reps calls (default 5) after one untimed call that loads the kernels.  `differing_pixels`
counts the pixels of the display buffer after the call that differ from render_into at the count each pixel reached (the
contract says 0).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCENES = [("irreg_1000", "irreg", 1000), ("random1M_2000", "random", 2000)]
SEED_SPP = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    only = set(filter(None, args.only.split(",")))
    ctx = R.Context(device=0)
    records = {}
    for key, name, size in SCENES:
        if only and key not in only:
            continue
        sc = ctx.scene_random(1 << 20, 1) if name == "random" else ctx.scene(name)
        pr = ctx.prepare_scene(size, size, sc)
        dev = torch.device("cuda", 0)
        frames = {}

        def frame(n):   # render_into's pixels at n samples
            if n not in frames:
                frames[n] = torch.empty((size, size), dtype=torch.int32, device=dev)
                torch.cuda.synchronize()
                ctx.render_into(frames[n].data_ptr(), size, size, pr, spp=n)
                ctx.sync()
            return frames[n]

        seed_acc = torch.empty((size, size, 3), dtype=torch.float32, device=dev)
        seed_rgb = torch.empty((size, size, 3), dtype=torch.float32, device=dev)
        seed_pix = torch.empty((size, size), dtype=torch.int32, device=dev)
        ctx.render_accumulate_into(seed_acc.data_ptr(), size, size, pr, 0, SEED_SPP, seed_pix.data_ptr(), seed_rgb.data_ptr())
        acc8 = torch.empty_like(seed_acc)
        rgb8 = torch.empty_like(seed_rgb)
        ctx.render_accumulate_into(acc8.data_ptr(), size, size, pr, 0, 2 * SEED_SPP, None, rgb8.data_ptr())
        ctx.sync()
        change = (rgb8 - seed_rgb).abs().sum(2)
        del acc8, rgb8

        g = torch.Generator(device=dev).manual_seed(7)
        rand = torch.rand((size, size), device=dev, generator=g)
        block = torch.zeros((size, size), dtype=torch.bool, device=dev)
        side = int(size * 0.1 ** 0.5) // 8 * 8           # whole tiles: multiples of 8 columns and 4 rows
        block[(size - side) // 8 * 4:(size - side) // 8 * 4 + side, (size - side) // 16 * 8:(size - side) // 16 * 8 + side] = True
        k = max(1, size * size // 10)
        top = torch.zeros(size * size, dtype=torch.bool, device=dev)
        top[torch.topk(change.flatten(), k).indices] = True
        masks = {"random_100": None, "random_50": rand < 0.5, "random_10": rand < 0.1, "random_1": rand < 0.01,
                 "tile_block_10": block, "largest_change_10": top.view(size, size),
                 "empty": torch.zeros((size, size), dtype=torch.bool, device=dev)}

        accum = torch.empty_like(seed_acc)
        counts = torch.empty((size, size), dtype=torch.int32, device=dev)
        pix = torch.empty_like(seed_pix)

        def reset():
            accum.copy_(seed_acc)
            counts.fill_(SEED_SPP)
            pix.copy_(seed_pix)
            torch.cuda.synchronize()

        def timed(call):
            reset()
            call()
            return ctx.last_render_ms()

        def accumulate():
            ctx.render_accumulate_into(accum.data_ptr(), size, size, pr, SEED_SPP, 2 * SEED_SPP, pix.data_ptr())

        timed(accumulate)
        acc_ms = statistics.median(timed(accumulate) for _ in range(args.reps))
        diff = int((pix != frame(2 * SEED_SPP)).sum())
        rec = {"size": size, "seed_spp": SEED_SPP, "accumulate_ms": round(acc_ms, 3), "accumulate_differing_pixels": diff}

        def adaptive(mask, n_add):
            ptr = None if mask is None else mask.data_ptr()
            return lambda: ctx.render_adaptive_into(accum.data_ptr(), counts.data_ptr(), size, size, pr, n_add, ptr, pix.data_ptr())

        work = [(m, 4) for m in masks] + [("random_10", 1)]
        for m, n_add in work:
            mask = masks[m]
            call = adaptive(mask, n_add)
            timed(call)
            ms = statistics.median(timed(call) for _ in range(args.reps))
            sel = torch.ones((size, size), dtype=torch.bool, device=dev) if mask is None else mask
            want = torch.where(sel, frame(SEED_SPP + n_add), frame(SEED_SPP))
            diff = int((pix != want).sum()) + int((counts != torch.where(sel, SEED_SPP + n_add, SEED_SPP)).sum())
            rec[f"{m}_add{n_add}"] = {"fraction": round(float(sel.float().mean()), 5), "ms": round(ms, 3),
                                      "vs_accumulate": round(ms / acc_ms, 4), "differing_pixels": diff}
            print(key, m, n_add, rec[f"{m}_add{n_add}"], file=sys.stderr, flush=True)
        records[key] = rec
        pr.free()
        sc.free()
        del frames, seed_acc, seed_rgb, seed_pix, accum, counts, pix, masks, rand, block, top, change
        torch.cuda.empty_cache()
    ctx.close()
    ok = all(v["differing_pixels"] == 0 for r in records.values() for v in r.values() if isinstance(v, dict))
    ok = ok and all(r["accumulate_differing_pixels"] == 0 for r in records.values())
    print(json.dumps({"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
                      "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "reps": args.reps, "workloads": records}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
