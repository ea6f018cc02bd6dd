"""Adaptive progressive rendering (include/ray_b200.h ray_b200_render_adaptive): samples added only to the pixels a mask
selects, each pixel continuing from its own sample count.  The contract is exactness: after any sequence of calls on
zeroed counts, a pixel's sum is the sum render_accumulate(0, counts[p]) leaves there, bit for bit, and its pixel and float
pixel are render_into(spp = counts[p])'s; pixels a call does not select are neither read nor written.

On the CPU the arithmetic is pinned down with the oracle: ragged per-pixel chains of in-order f32 sums of the per-sample
path colours equal the oracle's render at each pixel's count.  On the GPU every chunking, sample path, plan and scene is
checked bit for bit (NaN-aware) against render_accumulate and render_into."""
import numpy as np
import pytest

import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from oracle import pyoracle as O
from ray_query_cases import PLANS, _dev, _np, _torch, bits_differ
from test_render_accumulate import (BOUNDARY_PLAN, SCENES, _chain, _ctx, _gpu_colours, _one_shot, frame_of, last_spread_spp,
                                    sequential_sum)
from test_staging_plans import FORCED_PLANS, H, W, check_frame, expect, forced, variant  # noqa: F401 (forced: fixture)

SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes
INT32_MAX = 2 ** 31 - 1


def ragged_model(colours, masks, n_adds, accum=None, counts=None):
    """The contract on the CPU: colours [h, w, S, 3]; per call, every selected pixel with a valid count c gets samples
    [c, c + n) added in order.  Returns (accum, counts)."""
    h, w = colours.shape[:2]
    acc = np.zeros((h, w, 3), np.float32) if accum is None else accum.copy()
    cnt = np.zeros((h, w), np.int64) if counts is None else counts.astype(np.int64)
    for mask, n in zip(masks, n_adds):
        sel = np.ones((h, w), bool) if mask is None else mask.astype(bool)
        sel &= (cnt >= 0) & (cnt <= INT32_MAX - n)
        for c in np.unique(cnt[sel]):
            p = sel & (cnt == c)
            acc[p] = sequential_sum(colours[p], int(c), int(c) + n, acc[p])
        cnt[sel] += n
    return acc, cnt.astype(np.int32)


def random_masks(h, w, calls, seed, density=0.5):
    rng = np.random.default_rng(seed)
    return [rng.random((h, w)) < density for _ in range(calls)]


# ------------------------------------------------------------------------------------------ CPU: the arithmetic


@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "rgbbox_negative"])
def test_ragged_oracle_chains_equal_the_oracle_render(R, scene):
    h, w = 40, 56
    n_adds = [1, 3, 2, 1, 4]
    S = sum(n_adds)
    s, c = SCENES[scene]()
    o = Q.prepare_custom(s, c, h, w)
    colours = o.trace_paths(R.camera_rays(o.camera(), h, w, S).reshape(-1, 6))[0].reshape(h, w, S, 3)
    masks = random_masks(h, w, len(n_adds), 5, 0.6)
    masks[1] = None
    acc, cnt = ragged_model(colours, masks, n_adds)
    assert len(np.unique(cnt)) >= 4, "the chain is there to leave many different counts"
    prepared = O.Scene.custom(s, c).prepare(h, w)
    for n in np.unique(cnt):
        p = cnt == n
        if n == 0:
            continue
        want_pix, want_rgb, _ = prepared.render(h, w, int(n), want_rgb=True)
        pix, rgb = frame_of(acc[p], int(n))
        assert (pix == want_pix[p]).all(), n
        assert bits_differ(rgb, want_rgb[p]) == 0, n
        assert bits_differ(acc[p], sequential_sum(colours[p], 0, int(n))) == 0, n


def test_python_argument_checks(R):
    """Wrong devices, dtypes, shapes and layouts raise ValueError before anything reaches the library."""
    torch = _torch()

    class NoContext:
        device = 0

    h, w = 6, 10
    accum, counts = torch.zeros((h, w, 3)), torch.zeros((h, w), dtype=torch.int32)
    for bad in (accum, np.zeros((h, w, 3), np.float32), None, accum[:, :, :2]):
        with pytest.raises(ValueError):
            R.Context.render_adaptive(NoContext(), None, bad, counts, 1)
    if not torch.cuda.is_available():
        return
    a = torch.zeros((h, w, 3), device="cuda")
    c = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    m = torch.ones((h, w), dtype=torch.bool, device="cuda")
    good = dict(accum=a, counts=c, mask=m)
    bad_cases = [
        dict(accum=a.double()), dict(accum=a.transpose(0, 1)), dict(accum=a[:, :, :2]), dict(accum=a.reshape(h, w * 3)),
        dict(counts=c.cpu()), dict(counts=c.long()), dict(counts=c[:, :-1]), dict(counts=c.t()),
        dict(mask=m.cpu()), dict(mask=m.float()), dict(mask=m[:-1]), dict(mask=m.t()),
        dict(pixels=torch.zeros((h, w), device="cuda")), dict(pixels=torch.zeros((h, w + 1), dtype=torch.int32, device="cuda")),
        dict(rgb=torch.zeros((h, w, 3), dtype=torch.int32, device="cuda")), dict(rgb=torch.zeros((h, w, 3))),
    ]
    for change in bad_cases:
        args = dict(good, **change)
        with pytest.raises(ValueError):
            R.Context.render_adaptive(NoContext(), None, args.pop("accum"), args.pop("counts"), 1, **args)


# ------------------------------------------------------------------------------------------ GPU helpers


def _adaptive_chain(ctx, pr, h, w, masks, n_adds, accum=None, counts=None, check_untouched=False, plans=None):
    """Runs render_adaptive once per (mask, n_add) on one set of buffers (NaN-filled sums, zero counts, sentinel outputs
    unless given).  With check_untouched, asserts after every call that the pixels it did not select kept all four
    values.  Appends each call's plan to `plans` where given.  Returns numpy (accum, counts, pixels, rgb)."""
    torch = _torch()
    accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda") if accum is None else accum
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda") if counts is None else counts
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    for mask, n in zip(masks, n_adds):
        before = [t.clone() for t in (accum, counts, pix, rgb)] if check_untouched else None
        m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else torch.from_numpy(np.asarray(mask, bool)).cuda())
        ctx.render_adaptive(pr, accum, counts, n, mask=m, pixels=pix, rgb=rgb)
        assert ctx.last_plan()["query"] == "adaptive"
        if plans is not None:
            plans.append(ctx.last_plan())
        if check_untouched and m is not None:
            off = ~m.bool()
            for t0, t in zip(before, (accum, counts, pix, rgb)):
                assert torch.equal(t0.view(torch.int32)[off], t.view(torch.int32)[off]), "an unselected pixel changed"
    return _np(accum), _np(counts), _np(pix), _np(rgb)


def _check_counts_against_frames(ctx, pr, h, w, acc, cnt, pix, rgb, what):
    """Every pixel at count n > 0 equals render_into(spp = n) and render_accumulate(0, n)'s sum there."""
    ns = [int(n) for n in np.unique(cnt) if n > 0]
    for n in ns:
        p = cnt == n
        want_pix, want_rgb = _one_shot(ctx, pr, h, w, n)
        want_acc = _chain(ctx, pr, h, w, [(0, n)])[0]
        assert (pix[p] == want_pix[p]).all(), f"{what}: count {n}: {(pix[p] != want_pix[p]).sum()} pixels differ"
        assert bits_differ(rgb[p], want_rgb[p]) == 0, f"{what}: count {n}: float framebuffer"
        assert bits_differ(acc[p], want_acc[p]) == 0, f"{what}: count {n}: sums"
    return ns


# ------------------------------------------------------------------------------------------ GPU: identity with render_accumulate


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(1000, 1000), (37, 53), (4, 8)])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg"])
def test_uniform_counts_equal_render_accumulate(R, scene, h, w):
    """Mask NULL or all ones, every count at s_begin: each call is render_accumulate(s_begin, s_begin + n_add)."""
    torch = _torch()
    ctx, pr = _ctx(R, scene, h, w)
    ones = torch.ones((h, w), dtype=torch.bool, device="cuda")
    for split in ([(0, 64)], [(s, s + 1) for s in range(16)], [(0, 1), (1, 3), (3, 10), (10, 64)]):
        want = _chain(ctx, pr, h, w, split)
        masks = [None if k % 2 == 0 else ones for k in range(len(split))]
        acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, masks, [b - a for a, b in split])
        assert (cnt == split[-1][1]).all(), split
        assert bits_differ(acc, want[0]) == 0, f"{split}: sums"
        assert (pix == want[1]).all() and bits_differ(rgb, want[2]) == 0, f"{split}: frame"
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [1, 0])
def test_both_sample_paths(R, spread):
    """Calls of 1 (pixel-bound), 2 up to the last count whose finished-sample buffer fits the budget at 32 warps on this
    GPU's SMs (spread) and one more (pixel-bound); with wq_spread 0 all pixel-bound."""
    h, w = 4, 8
    last = last_spread_spp(_torch().cuda.get_device_properties(0).multi_processor_count)
    split = [(0, 1), (1, 3), (3, 10), (10, 11), (11, 75), (75, 75 + last), (75 + last, 76 + 2 * last)]
    ctx, pr = _ctx(R, "irreg", h, w, wq_spread=spread, **BOUNDARY_PLAN)
    want = _chain(ctx, pr, h, w, split)
    plans = []
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, [None] * len(split), [b - a for a, b in split], plans=plans)
    assert (cnt == split[-1][1]).all()
    assert bits_differ(acc, want[0]) == 0 and (pix == want[1]).all() and bits_differ(rgb, want[2]) == 0
    assert [p["spread"] for p in plans] == [int(spread and 1 < b - a <= last) for a, b in split]
    assert plans[-2]["spread"] == spread and plans[-1]["spread"] == 0 and {p["warps"] for p in plans} == {32}
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS + [{"wq_packet": 24}, {"wq_packet": 0}], ids=str)
def test_every_plan(R, plan):
    h, w = 203, 301
    masks, n_adds = random_masks(h, w, 3, 11), [1, 4, 11]
    ctx, pr = _ctx(R, "irreg", h, w, **plan)
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, masks, n_adds)
    ref, pr0 = _ctx(R, "irreg", h, w)
    assert len(_check_counts_against_frames(ref, pr0, h, w, acc, cnt, pix, rgb, str(plan))) >= 6
    ref.close()
    ctx.close()


@pytest.mark.gpu
def test_forced_boundaries(R, forced):
    """Every stage_cap point at K = 1 / 2, spread samples or not, with and without the packet walk: a one-sample call on
    half the pixels, then a two-sample call on all of them, against the oracle's frames at 1, 2 and 3 samples; the
    launched kAdaptive instantiations are exactly the 24 reachable ones."""
    torch = _torch()
    case, launched = forced["case"], set()
    half = torch.from_numpy(random_masks(H, W, 1, 3)[0]).cuda()
    for cap_name, cap, nodes, spheres in forced["caps"]:
        for plan in FORCED_PLANS:
            for packet in (0, 8):
                for spread in (1, 0):
                    what = f"{cap_name} (stage_cap {cap}), {plan}, wq_packet {packet}, wq_spread {spread}"
                    want = dict(kernel=R.KERNELS["warpqueue"], query="adaptive", k=plan["wq_k"], warps=plan["wq_warps"],
                                packet=packet, smem_nodes=nodes, smem_spheres=spheres)
                    with R.Context(device=0, stage_cap=cap, wq_packet=packet, wq_spread=spread, **plan) as ctx:
                        pr = case.prepare(ctx)
                        accum = torch.full((H, W, 3), float("nan"), dtype=torch.float32, device="cuda")
                        counts = torch.zeros((H, W), dtype=torch.int32, device="cuda")
                        pix = torch.full((H, W), SENTINEL, dtype=torch.int32, device="cuda")
                        rgb = torch.full((H, W, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
                        for mask, n in ((half, 1), (None, 2)):
                            ctx.render_adaptive(pr, accum, counts, n, mask=mask, pixels=pix, rgb=rgb)
                            p = ctx.last_plan()
                            expect(p, f"{what}, n_add {n}", spread=int(spread and n > 1), **want)
                            launched.add(variant(p))
                            cnt = _np(counts)
                            for c in np.unique(cnt[cnt > 0]):
                                sel = cnt == c
                                check_frame((_np(pix)[sel], _np(rgb)[sel]),
                                            (forced["frames"][int(c)][0][sel], forced["frames"][int(c)][1][sel]), f"{what}, count {c}")
                                if c > 1:
                                    assert bits_differ(_np(accum)[sel], forced["sums"][int(c)][sel]) == 0, f"{what}: sums"
    reachable = {("adaptive", False, k, sp, pk, st) for k in (1, 2) for sp in (False, True) for pk in (False, True)
                 for st in ("partial", "nodes", "whole")}
    missing = reachable - launched
    assert not missing, f"kAdaptive instantiations no case launched: {sorted(missing)}"
    assert launched == reachable and len(reachable) == 24


# ------------------------------------------------------------------------------------------ GPU: ragged chains, counts


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "random"])
def test_ragged_chains(R, scene):
    """Random masks per call: every distinct final count n has render_into(spp = n)'s pixels and render_accumulate(0, n)'s
    sums; a pixel a call does not select keeps all four values through that call, and a pixel no call selects keeps the
    sentinels."""
    h, w = 150, 211
    if scene == "random":
        ctx = R.Context(device=0)
        pr = ctx.prepare_scene(h, w, ctx.scene_random(30000, 1))
    else:
        ctx, pr = _ctx(R, scene, h, w)
    masks = random_masks(h, w, 6, 21, 0.4)
    never = np.zeros((h, w), bool)
    never[10:30, 40:90] = True
    for m in masks:
        m &= ~never
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, masks, [1, 2, 5, 1, 3, 2], check_untouched=True)
    assert (cnt[never] == 0).all() and (pix[never] == SENTINEL).all()
    assert (rgb.view(np.int32)[never] == SENTINEL).all() and np.isnan(acc[never]).all()
    assert len(_check_counts_against_frames(ctx, pr, h, w, acc, cnt, pix, rgb, scene)) >= 8
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_add", [1, 4])
def test_caller_supplied_sums_and_counts(R, n_add):
    """The result is f32 arithmetic on whatever accum holds at each pixel's count: random floats, +-0, +-inf and NaN."""
    torch = _torch()
    h, w = 37, 53
    ctx, pr = _ctx(R, "rgbbox_negative", h, w)
    rng = np.random.default_rng(n_add)
    start_counts = rng.integers(1, 7, (h, w)).astype(np.int32)
    colours = _gpu_colours(R, ctx, pr, h, w, int(start_counts.max()) + n_add)
    start = rng.standard_normal((h, w, 3)).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, (h, w, 3))
    special = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan])
    pick = rng.random((h, w, 3)) < 0.3
    start[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    mask = rng.random((h, w)) < 0.7
    want_acc, want_cnt = ragged_model(colours, [mask], [n_add], start, start_counts)
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, [mask], [n_add], _dev(start).reshape(h, w, 3),
                                         torch.from_numpy(start_counts).cuda())
    assert bits_differ(acc, want_acc) == 0 and (cnt == want_cnt).all()
    for n in np.unique(want_cnt[mask]):
        p = mask & (want_cnt == n)
        want_pix, want_rgb = frame_of(want_acc[p], int(n))
        assert (pix[p] == want_pix).all() and bits_differ(rgb[p], want_rgb) == 0, n
    assert (pix[~mask] == SENTINEL).all() and (cnt[~mask] == start_counts[~mask]).all()
    ctx.close()


@pytest.mark.gpu
def test_invalid_counts_and_empty_masks_write_nothing(R):
    torch = _torch()
    h, w, n_add = 37, 53, 3
    ctx, pr = _ctx(R, "irreg", h, w)
    rng = np.random.default_rng(2)
    bad = np.int32([-1, -(2 ** 31), -7, INT32_MAX, INT32_MAX - n_add + 1, INT32_MAX - 1])
    counts = np.zeros((h, w), np.int32)
    invalid = rng.random((h, w)) < 0.3
    counts[invalid] = bad[rng.integers(0, len(bad), int(invalid.sum()))]
    edge = ~invalid & (rng.random((h, w)) < 0.05)      # the largest valid count
    counts[edge] = INT32_MAX - n_add
    sentinel_acc = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, [None], [n_add], sentinel_acc, torch.from_numpy(counts).cuda())
    assert (cnt[invalid] == counts[invalid]).all() and (pix[invalid] == SENTINEL).all()
    assert (acc.view(np.int32)[invalid] == SENTINEL).all() and (rgb.view(np.int32)[invalid] == SENTINEL).all()
    assert (cnt[edge] == INT32_MAX).all() and (pix[edge] != SENTINEL).all()
    zero = ~invalid & ~edge
    assert _check_counts_against_frames(ctx, pr, h, w, acc, np.where(zero, cnt, 0), pix, rgb, "valid") == [n_add]
    # an empty mask: two launches, nothing written
    fresh = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    n0 = ctx.launch_count()
    acc2, cnt2, pix2, rgb2 = _adaptive_chain(ctx, pr, h, w, [np.zeros((h, w), bool)], [n_add], fresh, torch.from_numpy(counts).cuda())
    assert ctx.launch_count() - n0 == 2
    assert (acc2.view(np.int32) == SENTINEL).all() and (cnt2 == counts).all()
    assert (pix2 == SENTINEL).all() and (rgb2.view(np.int32) == SENTINEL).all()
    ctx.close()


# ------------------------------------------------------------------------------------------ GPU: scenes and sizes


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["rgbbox_x255", "irreg_x255", "rgbbox_top_down", "rgbbox_negative"])
def test_out_of_range_scenes(R, scene):
    h, w = 37, 53
    ctx, pr = _ctx(R, scene, h, w)
    acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, random_masks(h, w, 4, 9, 0.6), [1, 2, 1, 5])
    ns = _check_counts_against_frames(ctx, pr, h, w, acc, cnt, pix, rgb, scene)
    n = ns[-1]
    o_pix, o_rgb, _ = O.Scene.custom(*SCENES[scene]()).prepare(h, w).render(h, w, n, want_rgb=True)
    p = cnt == n
    assert (pix[p] == o_pix[p]).all() and bits_differ(rgb[p], o_rgb[p]) == 0, "oracle"
    ctx.close()


@pytest.mark.gpu
def test_golden_frames_through_a_chain(R, golden):
    """Half the pixels, then the other half, one sample each: the golden one-sample frames."""
    for name, (pixels, meta) in golden.items():
        h, w = meta["shape"]
        ctx, pr = _ctx(R, name.split("_")[0], h, w)
        half = random_masks(h, w, 1, 4)[0]
        _, cnt, pix, _ = _adaptive_chain(ctx, pr, h, w, [half, ~half], [1, 1])
        assert (cnt == 1).all() and (pix == pixels).all(), name
        ctx.close()


@pytest.mark.gpu
def test_million_spheres(R):
    h = w = 512
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_random(1 << 20, 1))
        acc, cnt, pix, rgb = _adaptive_chain(ctx, pr, h, w, random_masks(h, w, 3, 6), [4, 4, 4])
        assert len(_check_counts_against_frames(ctx, pr, h, w, acc, cnt, pix, rgb, "1 M spheres")) == 3


@pytest.mark.gpu
def test_largest_frame_sparse_mask(R):
    """2^30 pixels, one in 4096 selected: list and sum offsets pass 2^32 bytes; sampled rows against render_into."""
    torch = _torch()
    h = w = 32768
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.irreg())
        g = torch.Generator(device="cuda").manual_seed(3)
        mask = torch.rand((h, w), device="cuda", generator=g) < 1 / 4096
        rows = [0, 1, h // 2, h - 2, h - 1]
        mask[rows, ::97] = True
        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
        for n in (1, 1):
            ctx.render_adaptive(pr, accum, counts, n, mask=mask, pixels=pix)
        assert int((counts == 2).sum()) == int(mask.sum()) and int((counts[~mask] != 0).sum()) == 0
        assert int((pix[~mask] != SENTINEL).sum()) == 0
        del accum
        want = torch.empty((h, w), dtype=torch.int32, device="cuda")
        ctx.render_into(want.data_ptr(), h, w, pr, spp=2)
        ctx.sync()
        m = mask[rows]
        assert torch.equal(pix[rows][m], want[rows][m])
        del pix, want, counts, mask
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ GPU: ordering, errors


@pytest.mark.gpu
def test_renders_around_a_chain_plan_and_launch_as_before(R):
    torch = _torch()
    h, w = 250, 250
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")

    def run(with_adaptive):
        ctx, pr = _ctx(R, "irreg", h, w)
        accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        mask = torch.from_numpy(random_masks(h, w, 1, 8)[0]).cuda()
        frames, launches, plans = [], [], []
        for spp in (1, 1, 4, 1, 4):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            launches.append(ctx.launch_count() - n0)
            plans.append(ctx.last_plan())
            frames.append(_np(out))
            if with_adaptive:
                for n in (1, 3, 1):
                    n0 = ctx.launch_count()
                    ctx.render_adaptive(pr, accum, counts, n, mask=mask)
                    assert ctx.launch_count() - n0 == 2, "a selection pass and the render kernel"
        ctx.close()
        return frames, launches, plans

    plain, adaptive = run(False), run(True)
    assert plain[1] == adaptive[1] and plain[2] == adaptive[2]
    assert plain[1][0] > 1 and plain[1][1] == 1, "the learned order is recorded by the first frame and used by the second"
    for a, b in zip(plain[0], adaptive[0]):
        assert (a == b).all()


@pytest.mark.gpu
def test_torch_stream_and_freeing_the_scene_in_flight(R):
    torch = _torch()
    h, w = 300, 400
    masks, n_adds = random_masks(h, w, 2, 13), [3, 5]
    ctx, pr = _ctx(R, "rgbbox", h, w)
    want = _adaptive_chain(ctx, pr, h, w, masks, n_adds)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        got = _adaptive_chain(ctx, pr, h, w, masks, n_adds)
    for a, b in zip(want, got):
        assert bits_differ(a.view(np.float32), b.view(np.float32)) == 0, "torch stream"
    ctx.set_stream(None)
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    dmasks = [torch.from_numpy(m).cuda() for m in masks]
    torch.cuda.synchronize()
    for m, n in zip(dmasks, n_adds):
        s, c = SCENES["rgbbox"]()
        pr2 = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        ctx.render_adaptive_into(accum.data_ptr(), counts.data_ptr(), h, w, pr2, n, m.data_ptr(), pix.data_ptr())
        pr2.free()          # while the call may still be in flight
    ctx.sync()
    assert (_np(counts) == want[1]).all() and (_np(pix) == want[2]).all()
    sel = want[1] > 0
    assert bits_differ(_np(accum)[sel], want[0][sel]) == 0
    ctx.close()


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w = 37, 53
    ctx, pr = _ctx(R, "rgbbox", h, w)
    want = _chain(ctx, pr, h, w, [(0, 3)])
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    pix = torch.empty((h, w), dtype=torch.int32, device="cuda")

    class Freed:
        handle = None

    cases = [
        (dict(n_add=0), "n_add must be >= 1"),
        (dict(n_add=-3), "n_add must be >= 1"),
        (dict(accum=None), "accum_dev is required"),
        (dict(counts=None), "counts_dev is required"),
        (dict(h=0), "bad image size"),
        (dict(w=65537), "bad image size"),
        (dict(prepared=Freed()), "invalid prepared scene"),
        (dict(shard=(1, 2)), "shard set"),
    ]
    for change, message in cases:
        args = dict(accum=accum.data_ptr(), counts=counts.data_ptr(), h=h, w=w, prepared=pr, n_add=3, shard=None)
        args.update(change)
        if args["shard"]:
            ctx.set_shard(*args["shard"])
        n0 = ctx.launch_count()
        with pytest.raises(R.RayError, match=message):
            ctx.render_adaptive_into(args["accum"], args["counts"], args["h"], args["w"], args["prepared"], args["n_add"],
                                     None, pix.data_ptr())
        assert ctx.launch_count() == n0
        ctx.set_shard(0, 1)
        counts.zero_()
        torch.cuda.synchronize()
        ctx.render_adaptive_into(accum.data_ptr(), counts.data_ptr(), h, w, pr, 3, None, pix.data_ptr())
        ctx.sync()
        assert bits_differ(_np(accum), want[0]) == 0 and (_np(pix) == want[1]).all() and (_np(counts) == 3).all(), message
    ctx.close()
