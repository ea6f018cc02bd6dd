"""Sample indices far from 0: the spp rule of include/ray_b200.h where its f32 arithmetic changes regime.

Sample s of a pixel is offset by ox_s = frac(f32(s) * 0.7548776662f) and oy_s = frac(f32(s) * 0.5698402909f).  The
library computes this twice: the host builds a table (sample_offsets) that frames, views, G-buffers, scene batches and
progressive chunks read, and the adaptive kinds compute each sample's offsets in the kernel from the pixel's own count.
Once f32(s) * c reaches 2^21 the offsets are quarters, then halves, and from 2^23 / c on they are 0; past 2^24 f32(s)
itself rounds, so neighbouring samples are the same ray, and the counts that scale a sum and divide in Welford's update
are inexact.

On the CPU the rule is restated in numpy for any int64 index and checked against the library's host table and camera
rays, its regime thresholds are found by search, and windows of consecutive indices around each threshold are shown to
tell the rule from an f64 product and from an off-by-one index.  On the GPU the windows are reached through adaptive
pixels' counts and progressive chunks' s_begin, without tracing the samples before them, and compared with the rule on
the oracle's path colours of the restated rays: the in-kernel offsets and the host table must agree bit for bit.  The
offset-table cache is driven past its eviction with frames in flight on both lanes, and the boundary between spread
and pixel-bound samples is derived from the SM count."""
import numpy as np
import pytest

import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ
from test_render_accumulate import BOUNDARY_PLAN, SCENES, frame_of, last_spread_spp, sequential_sum
from test_render_adaptive import INT32_MAX, SENTINEL
from test_render_adaptive_var import select_model
from test_render_gbuffer import differ, oracle_gbuffer
from test_render_views import poses
from test_scene_batch import random_batch

F = np.float32
CONSTANTS = {"x": F(0.7548776662), "y": F(0.5698402909)}
TABLE_CACHE = 32      # offset tables a context keeps before it evicts the oldest (ensure_offsets, api_render.cu)

# ------------------------------------------------------------------------------------------ the rule in numpy


def offsets_rule(s):
    """(ox, oy) float32 of int64 sample indices s (any shape): f32(s) times each constant in f32, floor, difference."""
    sf = np.asarray(s, np.int64).astype(F)
    a, b = sf * CONSTANTS["x"], sf * CONSTANTS["y"]
    return a - np.floor(a), b - np.floor(b)


def offsets_f64(s):
    """A wrong rule: the product, floor and difference in f64, rounded to f32 at the end."""
    sd = np.asarray(s, np.int64).astype(np.float64)
    a, b = sd * np.float64(CONSTANTS["x"]), sd * np.float64(CONSTANTS["y"])
    return (a - np.floor(a)).astype(F), (b - np.floor(b)).astype(F)


def offsets_next(s):
    """A wrong rule: sample s gets the offsets of sample s + 1."""
    return offsets_rule(np.asarray(s, np.int64) + 1)


def rays_rule(camera, h, w, j, i, s, offsets=offsets_rule):
    """Camera rays of sample s of pixel (row j, column i) of an h x w frame for int64 arrays j, i, s (broadcast):
    float32 [..., 6], with the same f32 operations in the same order as R.camera_rays and primary_ray."""
    c = np.asarray(camera, F).reshape(12)
    j, i, s = np.broadcast_arrays(np.asarray(j, np.int64), np.asarray(i, np.int64), np.asarray(s, np.int64))
    ox, oy = offsets(s)
    u = (i.astype(F) + ox) / F(w)
    v = ((F(h) - j.astype(F)) + oy) / F(h)
    out = np.empty(s.shape + (6,), F)
    out[..., 0:3] = c[0:3]
    for a in range(3):   # llc + u*horizontal + v*vertical - origin, per component, left to right
        out[..., 3 + a] = ((c[3 + a] + u * c[6 + a]) + v * c[9 + a]) - c[a]
    return out


def window_rays(camera, h, w, start, k, offsets=offsets_rule):
    """rays_rule of samples [start, start + k) of every pixel: float32 [h, w, k, 6]"""
    return rays_rule(camera, h, w, np.arange(h)[:, None, None], np.arange(w)[None, :, None],
                     start + np.arange(k)[None, None, :], offsets)


def first_index(pred, lo=0, hi=INT32_MAX):
    """The smallest s in (lo, hi] with pred(s), for a predicate that is False at lo and monotone (False, then True)."""
    assert not pred(lo) and pred(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo = mid
    return hi


# The first sample whose f32 product with each constant reaches 2^e: offsets are multiples of 2^(e - 23) from there on
THRESHOLDS = {(axis, e): first_index(lambda s, c=c, e=e: F(s) * c >= F(2.0 ** e))
              for axis, c in CONSTANTS.items() for e in (21, 22, 23)}
ZERO_FROM = max(THRESHOLDS["x", 23], THRESHOLDS["y", 23])      # both offsets are 0 from here on
ROUNDS_FROM = first_index(lambda s: np.spacing(F(s)) > 1)      # f32(s) == f32(s + 1) from here on

K = 16
WINDOWS = {f"2^{e}/c{axis}": (t - K // 2, K) for (axis, e), t in sorted(THRESHOLDS.items())}
WINDOWS.update({
    "2^24": ((1 << 24) - K // 2, K),
    "2^25": ((1 << 25) - K // 2, K),
    "2^30": ((1 << 30) - K // 2, K),
    "INT32_MAX-16": (INT32_MAX - 16, K),      # the last window: counts end at INT32_MAX
    "INT32_MAX-9": (INT32_MAX - 9, 8),        # the chunk [INT32_MAX - 9, INT32_MAX - 1)
})


# ------------------------------------------------------------------------------------------ CPU: premises


@pytest.mark.parametrize("spp", [1, 2, 64, 4096])
def test_rule_equals_the_host_table_and_camera_rays(R, spp):
    ox, oy = offsets_rule(np.arange(spp))
    table = R.host_sample_offsets(spp)
    assert bits_differ(table[:, 0], ox) == 0 and bits_differ(table[:, 1], oy) == 0
    assert ox[0] == 0 and oy[0] == 0
    h, w = 13, 21
    cam = Q.prepare("irreg", h, w).camera()
    k = min(spp, 64)
    assert bits_differ(R.camera_rays(cam, h, w, spp)[:, :, :k], window_rays(cam, h, w, 0, k)) == 0


@pytest.mark.parametrize("axis,e", sorted(THRESHOLDS))
def test_regime_thresholds(axis, e):
    """From the threshold on the offsets are multiples of 2^(e - 23); in the samples just before it, some are not."""
    t, c = THRESHOLDS[axis, e], CONSTANTS[axis]
    assert abs(t - 2.0 ** e / float(c)) <= 2, "the product reaches 2^e where 2^e / c says"
    quantum = F(2.0 ** (e - 23))
    pick = 0 if axis == "x" else 1
    above = offsets_rule(np.arange(t, t + K))[pick]
    below = offsets_rule(np.arange(t - K, t))[pick]
    assert (np.mod(above, quantum) == 0).all()
    assert (np.mod(below, quantum) != 0).any()
    if e == 23:
        assert (above == 0).all() and (below != 0).any()


def test_f32_index_rounding():
    """f32(s) is exact and distinct below 2^24; from there on neighbouring indices share one f32 value."""
    assert ROUNDS_FROM == 1 << 24
    s = np.arange(ROUNDS_FROM - K, ROUNDS_FROM)
    assert (s.astype(F).astype(np.int64) == s).all()
    assert F(ROUNDS_FROM) == F(ROUNDS_FROM + 1) and F(ROUNDS_FROM + 2) != F(ROUNDS_FROM + 1)
    assert ZERO_FROM < ROUNDS_FROM, "both offsets vanish before the index itself rounds"
    assert 1.10e7 < THRESHOLDS["x", 23] < 1.12e7 and 1.46e7 < THRESHOLDS["y", 23] < 1.48e7


def test_past_both_thresholds_is_the_sample_0_ray(R):
    h, w = 13, 21
    cam = Q.prepare("rgbbox", h, w).camera()
    one = R.camera_rays(cam, h, w, 1)
    for name, (start, k) in WINDOWS.items():
        rays = window_rays(cam, h, w, start, k)
        same = np.array([bits_differ(rays[:, :, t], one[:, :, 0]) == 0 for t in range(k)])
        idx = start + np.arange(k)
        assert (same[idx >= ZERO_FROM]).all(), name
        if (idx < ZERO_FROM).any():
            assert not same[idx < ZERO_FROM].all(), f"{name}: every sample below {ZERO_FROM} gives the sample-0 ray"


def test_windows_discriminate():
    """On the oracle's path colours of a 4 x 8 frame, an f64 product differs from the rule in every window, and an
    off-by-one index in every window that starts below ZERO_FROM; past it every sample is the sample-0 ray, so no index
    model can be told apart there."""
    h, w = 4, 8
    o = Q.prepare("irreg", h, w)
    cam = o.camera()
    colours = lambda rays: o.trace_paths(rays.reshape(-1, 6))[0]
    for name, (start, k) in WINDOWS.items():
        want = colours(window_rays(cam, h, w, start, k))
        assert bits_differ(colours(window_rays(cam, h, w, start, k, offsets_f64)), want) > 0, f"{name}: f64 product"
        off_by_one = bits_differ(colours(window_rays(cam, h, w, start, k, offsets_next)), want)
        if start < ZERO_FROM:
            assert off_by_one > 0, f"{name}: s + 1"
        else:
            assert off_by_one == 0, name


# ------------------------------------------------------------------------------------------ the adaptive rule per window


def start_values(h, w, c, seed):
    """Finite caller-chosen start sums and M2 from 10^-2 up to about c, as if the pixel had c samples: some large
    enough that a sample is lost in rounding, some small enough that every bit of it counts."""
    rng = np.random.default_rng(seed)
    scale = F(10) ** rng.uniform(-2, np.log10(c), (h, w, 1)).astype(F)
    acc = rng.uniform(-1, 1, (h, w, 3)).astype(F) * scale
    m2 = rng.uniform(0, 1, (h, w, 3)).astype(F) * scale
    return acc, m2


def window_model(colours, c, acc, m2):
    """The adaptive rule for samples [c, c + k) of every pixel (colours [h, w, k, 3], c > 0) from the start sums acc and
    M2: the f32 sum in sample order, Welford's M2 += (x - S_n / f32(n)) (x - S_{n+1} / f32(n + 1)) for sample n, and the
    frame at c + k.  Returns (accum, m2, pixels, rgb)."""
    k = colours.shape[2]
    padded = np.concatenate([np.zeros_like(colours[:, :, :1]), colours], 2)   # sample c of the pixel at index 1
    acc_want = sequential_sum(padded, 1, k + 1, acc)
    a, m = acc.copy(), m2.copy()
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for t in range(k):
            x, n = colours[:, :, t], c + t
            nxt = a + x
            m = m + (x - a / F(n)) * (x - nxt / F(n + 1))
            a = nxt
    assert bits_differ(a, acc_want) == 0
    pix, rgb = frame_of(acc_want, c + k)
    return acc_want, m.astype(F), pix, rgb


# ------------------------------------------------------------------------------------------ GPU: windows


GPU_SCENES = ["rgbbox", "irreg", "random", "rgbbox_x255"]
SIZES = [(4, 8), (13, 21)]


def _scenes(ctx, name, h, w):
    """(GPU prepared scene, oracle prepared scene) of a scene of GPU_SCENES"""
    if name == "random":
        return ctx.prepare_scene(h, w, ctx.scene_random(1000, 1)), Q.prepare("random", h, w, n=1000, seed=1)
    if name in ("rgbbox", "irreg"):
        return ctx.prepare_scene(h, w, ctx.scene(name)), Q.prepare(name, h, w)
    s, c = SCENES[name]()
    return ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c)), Q.prepare_custom(s, c, h, w)


def _adaptive(ctx, pr, acc0, m20, c, n_adds, var):
    """render_adaptive (var: with M2) from every count at c and the start values, once per n_add: numpy (accum, m2 or
    None, counts, pixels, rgb) and each call's plan"""
    torch = _torch()
    h, w = acc0.shape[:2]
    accum = _dev(acc0)
    m2 = _dev(m20) if var else None
    counts = torch.full((h, w), c, dtype=torch.int32, device="cuda")
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    plans = []
    for n in n_adds:
        ctx.render_adaptive(pr, accum, counts, n, pixels=pix, rgb=rgb, m2=m2)
        plans.append(ctx.last_plan())
    return (_np(accum), _np(m2) if var else None, _np(counts), _np(pix), _np(rgb)), plans


def _check(got, want, what):
    acc, m2, cnt, pix, rgb = got
    w_acc, w_m2, w_cnt, w_pix, w_rgb = want
    assert bits_differ(acc, w_acc) == 0, f"{what}: accum, {bits_differ(acc, w_acc)} values differ"
    assert (cnt == w_cnt).all(), f"{what}: counts"
    assert (pix == w_pix).all(), f"{what}: {(pix != w_pix).sum()} pixels differ"
    assert bits_differ(rgb, w_rgb) == 0, f"{what}: float pixels"
    if m2 is not None:
        assert bits_differ(m2, w_m2) == 0, f"{what}: m2, {bits_differ(m2, w_m2)} values differ"


def _run_window(ctx, pr, colours, start, k, seed, spread, what):
    """Every way of reaching samples [start, start + k) of every pixel against the rule: adaptive and adaptive-var
    chains in one call and split, a progressive chunk, and the selection pass at the resulting counts."""
    torch = _torch()
    h, w = colours.shape[:2]
    acc0, m20 = start_values(h, w, start, seed)
    w_acc, w_m2, w_pix, w_rgb = window_model(colours, start, acc0, m20)
    want = (w_acc, w_m2, np.full((h, w), start + k, np.int32), w_pix, w_rgb)
    split = [1, 3, k - 4]
    for var in (False, True):
        for n_adds in ([k], split):
            got, plans = _adaptive(ctx, pr, acc0, m20, start, n_adds, var)
            tag = f"{what}, {'adaptive_var' if var else 'adaptive'} {n_adds}"
            _check(got, want, tag)
            assert [p["query"] for p in plans] == ["adaptive_var" if var else "adaptive"] * len(n_adds), tag
            assert [p["spread"] for p in plans] == [int(spread and n > 1) for n in n_adds], tag
    # the host table of the chunk against the in-kernel offsets of the adaptive kinds
    accum = _dev(acc0)
    pix, rgb = ctx.render_accumulate(pr, accum, start, start + k, want_rgb=True)
    p = ctx.last_plan()
    assert p["query"] == "accumulate" and p["spread"] == int(spread), what
    _check((_np(accum), None, want[2], _np(pix), _np(rgb)), want, f"{what}, render_accumulate")
    # the selection pass at these counts: f32(n) == f32(n - 1) past 2^24
    cnt, above = want[2], min(start + k + 1, INT32_MAX)
    for rule in ((0.02, 0.1, 2, INT32_MAX), (0.0, 0.0, 2, INT32_MAX), (1e-4, 0.0, start + k, above),
                 (0.1, 0.0, above, INT32_MAX), (0.1, 0.1, 2, start + k)):
        mask, n_sel = ctx.adaptive_select(_dev(w_acc), _dev(w_m2), torch.from_numpy(cnt).cuda(), *rule)
        sel, n = select_model(w_acc, w_m2, cnt, *rule)
        assert (_np(mask) == sel).all() and int(n_sel.item()) == n, f"{what}, select {rule}"


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("scene", GPU_SCENES)
def test_windows_against_the_rule(R, scene, h, w):
    """Every window under a spread plan and a pixel-bound one (wq_spread 0), from the same start values."""
    contexts = {spread: R.Context(device=0, wq_spread=spread) for spread in (1, 0)}
    prepared = {}
    for spread, ctx in contexts.items():
        prepared[spread], o = _scenes(ctx, scene, h, w)
    cam = o.camera()
    assert bits_differ(prepared[1].info()["camera"], cam) == 0
    for n, (name, (start, k)) in enumerate(WINDOWS.items()):
        colours = o.trace_paths(window_rays(cam, h, w, start, k).reshape(-1, 6))[0].reshape(h, w, k, 3)
        for spread, ctx in contexts.items():
            _run_window(ctx, prepared[spread], colours, start, k, n, spread, f"{scene} {h}x{w}, window {name}, spread {spread}")
    for ctx in contexts.values():
        ctx.close()


@pytest.mark.gpu
def test_selection_at_window_counts(R):
    """adaptive_select on counts drawn from every window, with M2 near the decision: the numpy rule bit for bit."""
    torch = _torch()
    h, w = 61, 67
    rng = np.random.default_rng(7)
    idx = np.concatenate([start + np.arange(k) for start, k in WINDOWS.values()])
    cnt = rng.choice(idx[idx >= 2], (h, w)).astype(np.int32)
    n = cnt.astype(np.int64)
    assert (n.astype(F) == (n - 1).astype(F)).any(), "some counts have f32(n) == f32(n - 1)"
    acc = (rng.uniform(0, 1, (h, w, 3)) * n[..., None]).astype(F)
    rel_err, floor = 0.01, 0.1
    mean = acc.sum(2).astype(np.float64) / n + floor
    target = (rel_err * mean) ** 2 * n * (n - 1.0)          # M2 summed over the channels at the decision
    m2 = (target[..., None] / 3 * rng.uniform(0.9, 1.1, (h, w, 3))).astype(F)
    with R.Context(device=0) as ctx:
        for rule in ((rel_err, floor, 2, INT32_MAX), (rel_err, floor, int(np.median(idx)), INT32_MAX),
                     (rel_err, floor, 2, int(np.median(idx)))):
            mask, n_sel = ctx.adaptive_select(_dev(acc), _dev(m2), torch.from_numpy(cnt).cuda(), *rule)
            sel, k = select_model(acc, m2, cnt, *rule)
            assert 0 < k < h * w, f"{rule}: the rule decides both ways"
            assert (_np(mask) == sel).all() and int(n_sel.item()) == k, f"{rule}: {(_np(mask) != sel).sum()} pixels differ"


# ------------------------------------------------------------------------------------------ GPU: the offset-table cache


def fifo_rebuilds(keys, capacity=TABLE_CACHE):
    """(distinct keys, how many times a key seen before had been evicted when it came back) for a cache of `capacity`
    entries that evicts the oldest"""
    cache, seen, rebuilt = [], set(), 0
    for key in keys:
        if key in cache:
            continue
        rebuilt += key in seen
        seen.add(key)
        if len(cache) >= capacity:
            cache.pop(0)
        cache.append(key)
    return len(seen), rebuilt


@pytest.mark.gpu
def test_offset_table_cache_eviction(R):
    """More than 32 distinct sample ranges on one context, then back to evicted ones, through every kind that reads the
    table, on two pipeline lanes, with nothing synchronised between the calls; every output against the oracle."""
    torch = _torch()
    h, w = 4, 8
    spheres, cam = O.Scene.named("irreg").arrays()
    cams = np.stack(poses(cam, 2, 3))
    bs, bcams = random_batch(2, 64, seed=3)
    oracles = {"frame": O.Scene.custom(spheres, cam).prepare(h, w), "view1": O.Scene.custom(spheres, cams[1]).prepare(h, w),
               "member0": O.Scene.custom(bs[0], bcams[0]).prepare(h, w), "member1": O.Scene.custom(bs[1], bcams[1]).prepare(h, w)}
    frames = {}

    def oracle(which, spp):
        if (which, spp) not in frames:
            frames[which, spp] = oracles[which].render(h, w, spp, want_rgb=True)[:2]
        return frames[which, spp]

    gb_oracle = Q.prepare_custom(spheres, cam, h, w)
    kinds = ["into", "batch", "pipeline", "views", "gbuffer", "scene_batch"]
    ops = [(kinds[n % len(kinds)], n) for n in range(1, 45)]                    # 44 distinct counts
    chain = [0, 45, 47, 50, 53, 57, 60, 64]                                      # every s_end a new count
    for q, (a, b) in enumerate(zip(chain[:-1], chain[1:])):
        ops.insert(6 * q + 3, ("chunk", (a, b)))
    ops += [(kinds[(n + 1) % len(kinds)], n) for n in range(1, 13)]              # back to evicted counts
    ops.append(("chunk", (0, 64)))
    keys = []
    for kind, n in ops:
        if kind == "chunk":
            keys.append(n)
        elif kind in ("batch", "pipeline"):
            keys += [(0, n), (0, 65 - n)]
        else:
            keys.append((0, n))
    distinct, rebuilt = fifo_rebuilds(keys)
    assert distinct > TABLE_CACHE and rebuilt >= 10, (distinct, rebuilt)

    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(spheres, cam))
        batch = ctx.prepare_scene_batch(h, w, _dev(bs), bcams)
        sentinel = lambda *shape: torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda")
        accums = [torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda") for _ in range(2)]
        outs = []
        for kind, n in ops:
            if kind in ("batch", "pipeline"):
                outs.append([(sentinel(h, w), sentinel(h, w, 3)) for _ in range(2)])
            elif kind == "views" or kind == "scene_batch":
                outs.append((sentinel(2, h, w), sentinel(2, h, w, 3)))
            elif kind == "gbuffer":
                outs.append({"id": sentinel(h, w), "depth": sentinel(h, w), "normal": sentinel(h, w, 3),
                             "albedo": sentinel(h, w, 3), "coverage": sentinel(h, w)})
            else:
                outs.append((sentinel(h, w), sentinel(h, w, 3)))
        torch.cuda.synchronize()
        for (kind, n), out in zip(ops, outs):
            if kind == "into":
                ctx.render_into(out[0].data_ptr(), h, w, pr, spp=n, out_rgb_dev=out[1].data_ptr())
            elif kind in ("batch", "pipeline"):
                ctx.set_pipeline(kind == "pipeline")
                ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=spp, out_dev=p.data_ptr(), out_rgb_dev=r.data_ptr())
                                  for spp, (p, r) in zip((n, 65 - n), out)])
            elif kind == "views":
                ctx.render_views_into(pr, cams, h, w, n, out[0].data_ptr(), out[1].data_ptr())
            elif kind == "gbuffer":
                ctx.render_gbuffer_into(pr, h, w, n, *[out[k].data_ptr() for k in ("id", "depth", "normal", "albedo", "coverage")])
            elif kind == "scene_batch":
                ctx.render_scene_batch_into(batch, h, w, n, out[0].data_ptr(), out[1].data_ptr())
            else:   # the chain on accums[0], the one call [0, 64) on accums[1]
                a, b = n
                ctx.render_accumulate_into(accums[int(n == (0, 64))].data_ptr(), h, w, pr, a, b, out[0].data_ptr(),
                                           out[1].data_ptr())
        ctx.set_pipeline(False)
        ctx.sync()
        f32 = lambda t: _np(t).view(np.float32)

        def frame_is(pix, rgb, want, what):
            assert (_np(pix) == want[0]).all(), f"{what}: {(_np(pix) != want[0]).sum()} pixels differ"
            assert bits_differ(f32(rgb), want[1]) == 0, f"{what}: float pixels"

        for (kind, n), out in zip(ops, outs):
            what = f"{kind} {n}"
            if kind == "into":
                frame_is(*out, oracle("frame", n), what)
            elif kind in ("batch", "pipeline"):
                for spp, (p, r) in zip((n, 65 - n), out):
                    frame_is(p, r, oracle("frame", spp), f"{what}: job at spp {spp}")
            elif kind == "views":
                for v, which in enumerate(("frame", "view1")):
                    frame_is(out[0][v], out[1][v], oracle(which, n), f"{what}: view {v}")
            elif kind == "scene_batch":
                for b, which in enumerate(("member0", "member1")):
                    frame_is(out[0][b], out[1][b], oracle(which, n), f"{what}: member {b}")
            elif kind == "gbuffer":
                got = {k: _np(v) if k in ("id", "coverage") else f32(v) for k, v in out.items()}
                differ(got, oracle_gbuffer(gb_oracle, spheres[:, 3:6], h, w, n), what)
            else:
                frame_is(*out, oracle("frame", n[1]), what)
        assert bits_differ(_np(accums[0]), _np(accums[1])) == 0, "the chain's sums are the one-call sums"


# ------------------------------------------------------------------------------------------ GPU: the spread boundary


@pytest.mark.gpu
def test_spread_boundary_of_every_frame_kind(R):
    """At 32 warps samples are spread up to the last count whose finished-sample buffer fits the budget on this GPU's
    SMs, and pixel-bound from the next one on: frames, chunks, views and scene batches, each against the oracle."""
    torch = _torch()
    h, w = 4, 8
    last = last_spread_spp(torch.cuda.get_device_properties(0).multi_processor_count)
    spheres, cam = O.Scene.named("irreg").arrays()
    bs, bcams = random_batch(2, 64, seed=4)
    want = {spp: O.Scene.custom(spheres, cam).prepare(h, w).render(h, w, spp, want_rgb=True)[:2] for spp in (last, last + 1)}
    want[2 * last + 1] = O.Scene.custom(spheres, cam).prepare(h, w).render(h, w, 2 * last + 1, want_rgb=True)[:2]

    def check(pix, rgb, spp, what, member=None):
        o = want[spp] if member is None else O.Scene.custom(bs[member], bcams[member]).prepare(h, w).render(h, w, spp, want_rgb=True)
        assert (_np(pix) == o[0]).all() and bits_differ(_np(rgb), o[1]) == 0, what

    with R.Context(device=0, **BOUNDARY_PLAN) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(spheres, cam))
        batch = ctx.prepare_scene_batch(h, w, _dev(bs), bcams)
        for spp, spread in ((last, 1), (last + 1, 0)):
            pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
            rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
            ctx.sync()
            p = ctx.last_plan()
            assert (p["query"], p["warps"], p["spread"]) == ("pixels", 32, spread), f"frame at spp {spp}: {p}"
            check(pix, rgb, spp, f"frame at spp {spp}")
            vp, vr = ctx.render_views(pr, np.stack([cam, cam]), h, w, spp, want_rgb=True)
            p = ctx.last_plan()
            assert (p["query"], p["warps"], p["spread"]) == ("views", 32, spread), f"views at spp {spp}: {p}"
            for v in range(2):
                check(vp[v], vr[v], spp, f"view {v} at spp {spp}")
            bp, br = ctx.render_scene_batch(batch, h, w, spp, want_rgb=True)
            p = ctx.last_plan()
            assert (p["query"], p["warps"], p["spread"]) == ("scene_batch", 32, spread), f"scene batch at spp {spp}: {p}"
            for b in range(2):
                check(bp[b], br[b], spp, f"member {b} at spp {spp}", member=b)
        accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        for (a, b), spread in (((0, last), 1), ((last, 2 * last + 1), 0)):
            pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
            p = ctx.last_plan()
            assert (p["query"], p["warps"], p["spread"]) == ("accumulate", 32, spread), f"chunk [{a}, {b}): {p}"
            check(pix, rgb, b, f"chunk [{a}, {b})")
