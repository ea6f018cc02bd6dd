#!/usr/bin/env python
"""Adaptive rendering driven by the noise estimate (include/ray_b200.h ray_b200_render_adaptive_var and
ray_b200_adaptive_select); prints one JSON line, and writes it to --out when given.

    python tools/bench_converge.py [--reps N] [--out FILE] [--only a,b,c]

(a) carry: what keeping M2 costs.  On bench_adaptive.py's scenes (irreg at 1000x1000, the 1 M-sphere scene at 2000x2000),
    seeded with 4 samples everywhere, one call of render_adaptive_var against the same call of render_adaptive: n_add 4 on
    100 % and 10 % random masks, and n_add 1 (the pixel-bound sample path) on 10 %.
(b) select: adaptive_select alone over a 2000x2000 frame of the 1 M-sphere scene at 8 samples.
(c) converge: render_converged (min_spp 8, step 8, max_spp 512) on irreg and on the 1 M-sphere scene at 1000x1000, at
    rel_err 0.02 and 0.01: total device time (the sum of every call's device time), mean spp, share of pixels at max_spp,
    and the RMSE of its float framebuffer against a high-spp render_into reference.  Against it, one uniform render_into
    at the same total sample count (the mean spp, rounded): its time and RMSE.

Times are device times, each the median of --reps runs (default 5) after one untimed run: the context's CUDA events
(ray_b200_context_last_render_ms) for the render calls, and torch CUDA events on the context's stream for
adaptive_select and for each call of the converged loop.  `differing_pixels` counts the pixels that differ from
render_into at the count each pixel reached (the contract says 0); for (c) the frames at every count come from one
render_accumulate chain in steps of 8 samples, which is bit for bit render_into at each step.  The card's name and power
limit are read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CARRY_SCENES = [("irreg_1000", "irreg", 1000), ("random1M_2000", "random", 2000)]
CONVERGE_SCENES = [("irreg_1000", "irreg", 1000, 4096), ("random1M_1000", "random", 1000, 1024)]   # (.., reference spp)
SEED_SPP = 4
MIN_SPP, STEP, MAX_SPP, MEAN_FLOOR = 8, 8, 512, 0.1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="a,b,c")
    args = ap.parse_args()
    import torch

    import raytracers_b200 as R

    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    parts = set(args.only.split(","))
    dev = torch.device("cuda", 0)
    ctx = R.Context(device=0)
    stream = torch.cuda.Stream(device=dev)
    ctx.set_stream(stream.cuda_stream)   # the context's launches go to a torch stream, so torch events can time them

    def scene(name):
        return ctx.scene_random(1 << 20, 1) if name == "random" else ctx.scene(name)

    def device_ms(call):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        call()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)

    def frame(pr, size, n):
        out = torch.empty((size, size), dtype=torch.int32, device=dev)
        stream.synchronize()
        ctx.render_into(out.data_ptr(), size, size, pr, spp=n)
        ctx.sync()
        return out

    out = {"gpu": gpu[0] if gpu else None, "power_limit_w": float(gpu[1]) if len(gpu) > 1 else None,
           "max_sm_clock_mhz": float(gpu[2]) if len(gpu) > 2 else None, "reps": args.reps}
    ok = True

    # ---------------------------------------------------------------------------------------- (a) the cost of M2
    if "a" in parts:
        carry = {}
        for key, name, size in CARRY_SCENES:
            sc = scene(name)
            pr = ctx.prepare_scene(size, size, sc)
            shape3 = (size, size, 3)
            seed_acc = torch.empty(shape3, dtype=torch.float32, device=dev)
            seed_m2 = torch.empty(shape3, dtype=torch.float32, device=dev)
            seed_cnt = torch.zeros((size, size), dtype=torch.int32, device=dev)
            seed_pix = torch.empty((size, size), dtype=torch.int32, device=dev)
            stream.synchronize()
            ctx.render_adaptive_var_into(seed_acc.data_ptr(), seed_m2.data_ptr(), seed_cnt.data_ptr(), size, size, pr, SEED_SPP,
                                         None, seed_pix.data_ptr())
            ctx.sync()
            g = torch.Generator(device=dev).manual_seed(7)
            rand = torch.rand((size, size), device=dev, generator=g)
            masks = {"random_100": None, "random_10": rand < 0.1}
            accum, m2 = torch.empty_like(seed_acc), torch.empty_like(seed_m2)
            counts, pix = torch.empty_like(seed_cnt), torch.empty_like(seed_pix)
            frames = {n: frame(pr, size, n) for n in (SEED_SPP, SEED_SPP + 1, 2 * SEED_SPP)}
            rec = {"size": size, "seed_spp": SEED_SPP}
            for m, n_add in (("random_100", 4), ("random_10", 4), ("random_10", 1)):
                mask = masks[m]
                mp = None if mask is None else mask.data_ptr()
                times = {}
                for var in (False, True):
                    def call():
                        if var:
                            ctx.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), size, size, pr,
                                                         n_add, mp, pix.data_ptr())
                        else:
                            ctx.render_adaptive_into(accum.data_ptr(), counts.data_ptr(), size, size, pr, n_add, mp,
                                                     pix.data_ptr())

                    def timed():
                        accum.copy_(seed_acc); m2.copy_(seed_m2); counts.copy_(seed_cnt); pix.copy_(seed_pix)
                        torch.cuda.synchronize()
                        call()
                        ctx.sync()
                        return ctx.last_render_ms()

                    timed()
                    times[var] = statistics.median(timed() for _ in range(args.reps))
                    sel = torch.ones((size, size), dtype=torch.bool, device=dev) if mask is None else mask
                    want = torch.where(sel, frames[SEED_SPP + n_add], frames[SEED_SPP])
                    diff = int((pix != want).sum()) + int((counts != torch.where(sel, SEED_SPP + n_add, SEED_SPP)).sum())
                    times[(var, "diff")] = diff
                    ok = ok and diff == 0
                rec[f"{m}_add{n_add}"] = {"adaptive_ms": round(times[False], 3), "adaptive_var_ms": round(times[True], 3),
                                          "var_vs_adaptive": round(times[True] / times[False], 4),
                                          "differing_pixels": times[(False, "diff")] + times[(True, "diff")]}
                print("a", key, m, n_add, rec[f"{m}_add{n_add}"], file=sys.stderr, flush=True)
            carry[key] = rec
            pr.free(); sc.free()
            del seed_acc, seed_m2, seed_cnt, seed_pix, accum, m2, counts, pix, frames, masks, rand
            torch.cuda.empty_cache()
        out["carry"] = carry

    # ---------------------------------------------------------------------------------------- (b) the selection pass
    if "b" in parts:
        size = 2000
        sc = scene("random")
        pr = ctx.prepare_scene(size, size, sc)
        acc = torch.empty((size, size, 3), dtype=torch.float32, device=dev)
        m2 = torch.empty_like(acc)
        cnt = torch.zeros((size, size), dtype=torch.int32, device=dev)
        mask = torch.empty((size, size), dtype=torch.bool, device=dev)
        n_sel = torch.empty(1, dtype=torch.int32, device=dev)
        stream.synchronize()
        ctx.render_adaptive_var_into(acc.data_ptr(), m2.data_ptr(), cnt.data_ptr(), size, size, pr, 8)
        ctx.sync()
        sel = {}
        for rel_err in (0.02, 0.01):
            call = lambda: ctx.adaptive_select_into(acc.data_ptr(), m2.data_ptr(), cnt.data_ptr(), size, size, rel_err,
                                                    MEAN_FLOOR, MIN_SPP, MAX_SPP - STEP + 1, mask.data_ptr(), n_sel.data_ptr())
            device_ms(call)
            ms = statistics.median(device_ms(call) for _ in range(max(args.reps, 20)))
            sel[f"rel_err_{rel_err}"] = {"ms": round(ms, 4), "selected_fraction": round(int(n_sel.item()) / size ** 2, 4),
                                         "gb_per_s": round((size * size * (3 * 4 * 2 + 4 + 1)) / (ms * 1e-3) / 1e9, 1)}
            print("b", rel_err, sel[f"rel_err_{rel_err}"], file=sys.stderr, flush=True)
        out["select_2000"] = sel
        pr.free(); sc.free()
        del acc, m2, cnt, mask
        torch.cuda.empty_cache()

    # ---------------------------------------------------------------------------------------- (c) the converged loop
    if "c" in parts:
        conv = {}
        for key, name, size, ref_spp in CONVERGE_SCENES:
            sc = scene(name)
            pr = ctx.prepare_scene(size, size, sc)
            shape3 = (size, size, 3)
            ref_rgb = torch.empty(shape3, dtype=torch.float32, device=dev)
            ref_pix = torch.empty((size, size), dtype=torch.int32, device=dev)
            stream.synchronize()
            ctx.render_into(ref_pix.data_ptr(), size, size, pr, spp=ref_spp, out_rgb_dev=ref_rgb.data_ptr())
            ctx.sync()
            rec = {"size": size, "reference_spp": ref_spp, "reference_ms": round(ctx.last_render_ms(), 1)}

            def rmse(rgb):
                return math.sqrt(float(((rgb.double() - ref_rgb.double()) ** 2).mean()))

            for rel_err in (0.02, 0.01):
                pix, rgb, counts, stats = ctx.render_converged(pr, size, size, rel_err, mean_floor=MEAN_FLOOR, min_spp=MIN_SPP,
                                                               step=STEP, max_spp=MAX_SPP, want_rgb=True)

                def loop():   # the loop render_converged runs, with every call timed on the device
                    acc = torch.empty(shape3, dtype=torch.float32, device=dev)
                    m2 = torch.empty(shape3, dtype=torch.float32, device=dev)
                    cnt = torch.zeros((size, size), dtype=torch.int32, device=dev)
                    mask = torch.empty((size, size), dtype=torch.bool, device=dev)
                    n_sel = torch.empty(1, dtype=torch.int32, device=dev)
                    stream.synchronize()
                    total = device_ms(lambda: ctx.render_adaptive_var_into(acc.data_ptr(), m2.data_ptr(), cnt.data_ptr(), size,
                                                                           size, pr, MIN_SPP))
                    while True:
                        total += device_ms(lambda: ctx.adaptive_select_into(
                            acc.data_ptr(), m2.data_ptr(), cnt.data_ptr(), size, size, rel_err, MEAN_FLOOR, MIN_SPP,
                            MAX_SPP - STEP + 1, mask.data_ptr(), n_sel.data_ptr()))
                        total += device_ms(lambda: ctx.render_adaptive_var_into(acc.data_ptr(), m2.data_ptr(), cnt.data_ptr(),
                                                                                size, size, pr, STEP, mask.data_ptr()))
                        if int(n_sel.item()) == 0:
                            break
                    return total, cnt

                loop()
                runs = [loop() for _ in range(args.reps)]
                ms = statistics.median(t for t, _ in runs)
                diff = sum(int((c != counts).sum()) for _, c in runs)   # the timed loop is render_converged's
                # the pixels against render_into at each count: one render_accumulate chain in steps of STEP
                top = int(counts.max())
                acc = torch.empty(shape3, dtype=torch.float32, device=dev)
                step_pix = torch.empty((size, size), dtype=torch.int32, device=dev)
                for s in range(0, top, STEP):
                    stream.synchronize()
                    ctx.render_accumulate_into(acc.data_ptr(), size, size, pr, s, s + STEP, step_pix.data_ptr())
                    ctx.sync()
                    here = counts == s + STEP
                    diff += int((pix[here] != step_pix[here]).sum())
                diff += int(((counts - MIN_SPP) % STEP != 0).sum()) + int((counts > MAX_SPP).sum())
                ok = ok and diff == 0
                mean_spp = float(counts.double().mean())
                uni_spp = max(1, round(mean_spp))
                uni_rgb = torch.empty(shape3, dtype=torch.float32, device=dev)
                uni_ms = []
                for _ in range(args.reps + 1):
                    stream.synchronize()
                    ctx.render_into(step_pix.data_ptr(), size, size, pr, spp=uni_spp, out_rgb_dev=uni_rgb.data_ptr())
                    ctx.sync()
                    uni_ms.append(ctx.last_render_ms())
                rec[f"rel_err_{rel_err}"] = {
                    "converged_ms": round(ms, 2), "rounds": stats["rounds"], "mean_spp": round(mean_spp, 2),
                    "at_max_spp": round(float((counts == MAX_SPP).double().mean()), 4), "rmse": rmse(rgb),
                    "uniform_spp": uni_spp, "uniform_ms": round(statistics.median(uni_ms[1:]), 2), "uniform_rmse": rmse(uni_rgb),
                    "differing_pixels": diff}
                print("c", key, rel_err, rec[f"rel_err_{rel_err}"], file=sys.stderr, flush=True)
                del acc, step_pix, uni_rgb, pix, rgb, counts
            conv[key] = rec
            pr.free(); sc.free()
            del ref_rgb, ref_pix
            torch.cuda.empty_cache()
        out["converge"] = conv

    ctx.set_stream(None)
    ctx.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
