#!/usr/bin/env python
"""Small renders that exercise every path of the default kernels (K3 warp-queue: item queues, packet walk, sample
spreading, pixel-bound samples, two frames in flight, compact shard layout, peer-frame flags; K5 lane-walk) for
compute-sanitizer (tools/sanitize.sh), then every entry point that writes device memory at the small sizes of
tests/test_memory_contract.py: frames and shards, batches, detile, accumulate, adaptive chains with adaptive_select,
views, every G-buffer subset, every ray query per-call and ranged, device-prepared scenes with update and read-back,
the learned claim order and the heavy-first probe.  Every result is checked against the oracle."""
import os
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import raytracers_b200 as R  # noqa: E402
from oracle import pyoracle as O  # noqa: E402


def check(got, want, what):
    bad = int((got != want).sum())
    print(f"{what}: {'ok' if bad == 0 else f'{bad} pixels differ'}", flush=True)
    return bad


def main():
    bad = 0
    h, w = 40, 72
    want = {(n, s): getattr(O.Scene, n)().prepare(h, w).render(h, w, spp=s)[0] for n in ("rgbbox", "irreg") for s in (1, 3)}
    for kernel, tuning in (("warpqueue", {}), ("warpqueue", dict(wq_packet=8)), ("warpqueue", dict(wq_spread=0)), ("warpqueue", dict(wq_low=40, wq_k=1)),
                           ("warpqueue", dict(wq_low=-1)), ("lanewalk", {})):
        with R.Context(kernel=kernel, **tuning) as ctx:
            prep = {n: ctx.prepare_scene(h, w, ctx.scene(n)) for n in ("rgbbox", "irreg")}
            for (n, s), wnt in want.items():
                bad += check(ctx.render_host(h, w, prep[n], spp=s), wnt, f"{kernel} {tuning} {n} spp={s}")
            # two frames in flight + the compact shard layout + peer-frame flags, device buffers from futhark_new_i32_2d
            lib = ctx.lib
            zeros = np.zeros((h, w), np.int32)
            imgs = [lib.futhark_new_i32_2d(ctx.handle, zeros.ctypes.data, h, w) for _ in range(3)]
            ptrs = [lib.futhark_values_raw_i32_2d(ctx.handle, im) for im in imgs]
            flags, _ = ctx.ipc_alloc(1024)
            jobs = [dict(prepared=prep["irreg"], h=h, w=w, spp=3, out_dev=ptrs[0], done_flag=flags),
                    dict(prepared=prep["rgbbox"], h=h, w=w, spp=1, out_dev=ptrs[1], done_flag=flags + 128),
                    dict(prepared=prep["rgbbox"], h=h, w=w, spp=3, out_dev=ptrs[2], wait_flag=flags, wait_value=1)]
            ctx.render_batch(jobs)
            ctx.flag_wait(flags + 128, 1)
            ctx.sync()
            for im, key in zip(imgs, (("irreg", 3), ("rgbbox", 1), ("rgbbox", 3))):
                out = np.empty((h, w), np.int32)
                lib.futhark_values_i32_2d(ctx.handle, im, out.ctypes.data)
                bad += check(out, want[key], f"{kernel} {tuning} batch {key}")
                lib.futhark_free_i32_2d(ctx.handle, im)
            bad += ctx.flag_timeouts()
            ctx.ipc_free(flags)
    with R.Context(kernel="warpqueue") as ctx:   # deep tree: global-memory nodes (256-bit loads), overflow guard of the node queue
        n, hh, ww = 30000, 32, 48
        wnt, _, _ = O.render_scene("random", hh, ww, n=n, seed=3)
        pr = ctx.prepare_scene(hh, ww, ctx.scene_random(n, 3))
        bad += check(ctx.render_host(hh, ww, pr), wnt, "warpqueue deep tree")
    # every node staged with the spheres read from global memory, and a whole scene of more than 2048 sphere records
    # (the staging copy's second 32 KB piece of them) behind 3 warps' queues
    for n, tuning, want_staged in ((600, dict(stage_cap=64 * 599), (599, 0)), (2600, dict(wq_warps=3), (2599, 2600))):
        hh, ww = 32, 48
        with R.Context(kernel="warpqueue", **tuning) as ctx:
            pr = ctx.prepare_scene(hh, ww, ctx.scene_random(n, 5))
            for s in (1, 3):
                wnt, _, _ = O.render_scene("random", hh, ww, spp=s, n=n, seed=5)
                bad += check(ctx.render_host(hh, ww, pr, spp=s), wnt, f"warpqueue {tuning} n={n} spp={s}")
                plan = ctx.last_plan()
                staged = (plan["smem_nodes"], plan["smem_spheres"])
                if staged != want_staged:
                    print(f"warpqueue {tuning} n={n} spp={s}: staged {staged}, expected {want_staged}", flush=True)
                    bad += 1
    bad += memory_contract_cases()
    print("SANITIZE_TARGET", "OK" if bad == 0 else f"FAILED ({bad})", flush=True)
    return 1 if bad else 0


def memory_contract_cases():
    """The cases of tests/test_memory_contract.py (guarded outputs, sentinel 0xFF), one small size each."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import test_memory_contract as M
    bad = 0

    def run(what, fn, *args):
        nonlocal bad
        try:
            fn(*args)
            print(f"{what}: ok", flush=True)
        except Exception:   # a failed check or an error of the call: counted, and the other cases still run
            bad += 1
            print(f"{what}: FAILED\n{traceback.format_exc()}", flush=True)
    e = M.Env(heavy_first=-1)
    try:
        for name, (h, w), spp in (("rgbbox", (9, 5), 3), ("irreg", (33, 65), 3), ("comb", (1, 37), 1), ("irreg", (37, 1), 16)):
            for case in M.FRAME_CASES:
                run(f"{case.__name__} {name} {h}x{w} spp={spp}", case, e, name, h, w, spp, 0xFF)
        for name in M.SCENE_NAMES:
            run(f"queries {name}", M.case_queries, e, name, 33, 0xFF, M.KS, 4)
            run(f"device scene {name}", M.case_scene_device, e, name, 0xFF)
        run("learned order and heavy-first frames", M._learned_order_frames, e, 0xFF)
    finally:
        e.close()
    return bad


if __name__ == "__main__":
    sys.exit(main())
