"""Progressive rendering (include/ray_b200.h ray_b200_render_accumulate): a frame's samples added to a running sum over
several calls.  The contract is exactness: any chain of calls [0, a), [a, b), ..., [y, S) leaves the same f32 sums as one
call [0, S), bit for bit, and its frame equals render_into(spp = S).

On the CPU the arithmetic is pinned down with the oracle: the in-order f32 sum of the per-sample colours of trace_paths,
carried between chunks with the rule for sample 0, scaled by 1/S and quantised, equals the oracle's render at S samples.
On the GPU every chunking, sample path, plan, shard and scene is checked bit for bit (NaN-aware) against the one-shot
frame and against the same sum of the GPU's own trace_paths colours."""
import numpy as np
import pytest

import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from oracle import pyoracle as O
from ray_query_cases import PLANS, _dev, _np, _torch, bits_differ, quantise

SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes
SPLITS = {
    "whole": [(0, 64)],
    "ones": [(s, s + 1) for s in range(64)],
    "uneven": [(0, 1), (1, 3), (3, 10), (10, 64)],
}


def random_split(total, seed, parts=6):
    cuts = sorted(np.random.default_rng(seed).choice(np.arange(1, total), parts - 1, replace=False).tolist())
    edges = [0] + cuts + [total]
    return list(zip(edges[:-1], edges[1:]))


def sequential_sum(colours, s_begin, s_end, start=None):
    """colours [..., S, 3] float32: start + colour_{s_begin} + ... + colour_{s_end-1} in sample order in f32; with
    s_begin == 0 the sum starts as colour_0 itself (start is ignored)."""
    acc = colours[..., 0, :].copy() if s_begin == 0 else np.asarray(start, np.float32) + colours[..., s_begin, :]
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(s_begin + 1, s_end):
            acc = acc + colours[..., s, :]
    return acc.astype(np.float32)


def frame_of(acc, s_end):
    """(pixels, rgb) of a frame from its sum over s_end samples: scaled by 1/s_end in f32 (1 * x = x at s_end = 1)."""
    with np.errstate(invalid="ignore", over="ignore"):
        rgb = (np.float32(1) / np.float32(s_end)) * np.asarray(acc, np.float32)
    return quantise(rgb), rgb


# ------------------------------------------------------------------------------------------ scenes


def _builtin(name):
    return O.Scene.named(name).arrays()


def _recolour(name, f):
    s, c = _builtin(name)
    s = s.copy()
    s[:, 3:6] = f(s[:, 3:6])
    return s, c


def _camera(name, look_from, look_at):
    s, c = _builtin(name)
    c = c.copy()
    c[0:3], c[3:6] = look_from, look_at
    return s, c


SCENES = {
    "rgbbox": lambda: _builtin("rgbbox"),
    "irreg": lambda: _builtin("irreg"),
    "rgbbox_negative": lambda: _recolour("rgbbox", lambda col: col * np.float32(-255)),   # -0.0 sums
    "rgbbox_x255": lambda: _recolour("rgbbox", lambda col: col * np.float32(255)),
    "irreg_x255": lambda: _recolour("irreg", lambda col: col * np.float32(255)),
    "rgbbox_top_down": lambda: _camera("rgbbox", (0, 40, 0), (0, 0, 0)),                  # NaN camera rays
}


# ------------------------------------------------------------------------------------------ CPU: the arithmetic


@pytest.mark.parametrize("spp", [1, 7, 16])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "rgbbox_negative"])
def test_chunked_oracle_sums_equal_the_oracle_render(R, scene, spp):
    h, w = 40, 56
    s, c = SCENES[scene]()
    o = Q.prepare_custom(s, c, h, w)
    rays = R.camera_rays(o.camera(), h, w, spp).reshape(-1, 6)
    colours = o.trace_paths(rays)[0].reshape(h, w, spp, 3)
    want_pix, want_rgb, _ = O.Scene.custom(s, c).prepare(h, w).render(h, w, spp, want_rgb=True)
    if scene == "rgbbox_negative":
        assert (np.signbit(colours) & (colours == 0)).any(), "the scene is there to produce -0.0 colours"
    splits = [[(0, spp)], [(k, k + 1) for k in range(spp)]] + ([random_split(spp, spp, min(spp, 4))] if spp > 1 else [])
    for split in splits:
        acc = None
        for a, b in split:
            acc = sequential_sum(colours, a, b, acc)
        pix, rgb = frame_of(acc, spp)
        assert bits_differ(acc, sequential_sum(colours, 0, spp)) == 0, split
        assert (pix == want_pix).all(), split
        assert bits_differ(rgb, want_rgb) == 0, split


def test_a_sum_of_means_is_not_the_frame(R):
    """Why the library carries the sum: the mean of separate renders differs from the frame in some pixels."""
    h, w, spp = 40, 56, 16
    o = Q.prepare("irreg", h, w)
    colours = o.trace_paths(R.camera_rays(o.camera(), h, w, spp).reshape(-1, 6))[0].reshape(h, w, spp, 3)
    halves = (sequential_sum(colours, 0, 8) * np.float32(1 / 8) + sequential_sum(colours[..., 8:, :], 0, 8) * np.float32(1 / 8))
    assert bits_differ(halves * np.float32(0.5), frame_of(sequential_sum(colours, 0, spp), spp)[1]) > 0


# ------------------------------------------------------------------------------------------ GPU helpers


def _ctx(R, scene, h, w, **kw):
    ctx = R.Context(device=0, **kw)
    sc = ctx.scene(scene) if scene in ("rgbbox", "irreg") else ctx.scene_from_arrays(*SCENES[scene]())
    return ctx, ctx.prepare_scene(h, w, sc)


def _one_shot(ctx, pr, h, w, spp):
    torch = _torch()
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb)


def _chain(ctx, pr, h, w, split, accum=None):
    """Runs the calls of `split` on one accum buffer (NaN-filled unless given: sample 0 must not read it)."""
    torch = _torch()
    if accum is None:
        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
    pix = rgb = None
    for a, b in split:
        pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
    return _np(accum), _np(pix), _np(rgb)


def _gpu_colours(R, ctx, pr, h, w, spp):
    rays = R.camera_rays(pr.info()["camera"], h, w, spp).reshape(-1, 6)
    return _np(ctx.trace_paths(pr, _dev(rays))[0]).reshape(h, w, spp, 3)


def _check_against(acc, pix, rgb, want_acc, want_pix, want_rgb, what):
    assert bits_differ(acc, want_acc) == 0, f"{what}: accum"
    assert (pix == want_pix).all(), f"{what}: {(pix != want_pix).sum()} pixels differ"
    assert bits_differ(rgb, want_rgb) == 0, f"{what}: float framebuffer"


# ------------------------------------------------------------------------------------------ GPU: exactness


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(1000, 1000), (37, 53), (4, 8)])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg"])
def test_every_chunking_equals_one_render(R, scene, h, w):
    S = 64
    ctx, pr = _ctx(R, scene, h, w)
    want_pix, want_rgb = _one_shot(ctx, pr, h, w, S)
    splits = dict(SPLITS, random=random_split(S, h * w))
    whole = _chain(ctx, pr, h, w, splits["whole"])
    if h * w <= 4096:
        colours = _gpu_colours(R, ctx, pr, h, w, S)
        assert bits_differ(whole[0], sequential_sum(colours, 0, S)) == 0
    for name, split in splits.items():
        acc, pix, rgb = _chain(ctx, pr, h, w, split)
        _check_against(acc, pix, rgb, whole[0], want_pix, want_rgb, name)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 4])
def test_caller_supplied_sums(R, chunk):
    """With s_begin > 0 the result is f32 arithmetic on whatever accum holds: random floats, +-0, +-inf and NaN."""
    torch = _torch()
    h, w, s_begin = 37, 53, 5
    s_end = s_begin + chunk
    ctx, pr = _ctx(R, "rgbbox_negative", h, w)
    colours = _gpu_colours(R, ctx, pr, h, w, s_end)
    rng = np.random.default_rng(chunk)
    start = rng.standard_normal((h, w, 3)).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, (h, w, 3))
    special = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan])
    pick = rng.random((h, w, 3)) < 0.3
    start[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    accum = _dev(start).reshape(h, w, 3)
    acc, pix, rgb = _chain(ctx, pr, h, w, [(s_begin, s_end)], accum)
    want = sequential_sum(colours, s_begin, s_end, start)
    want_pix, want_rgb = frame_of(want, s_end)
    _check_against(acc, pix, rgb, want, want_pix, want_rgb, "seeded")
    # s_begin == 0 ignores what the buffer holds
    for fill in (float("nan"), float("inf"), -0.0):
        accum = torch.full((h, w, 3), fill, dtype=torch.float32, device="cuda")
        acc, _, _ = _chain(ctx, pr, h, w, [(0, s_end)], accum)
        assert bits_differ(acc, sequential_sum(colours, 0, s_end)) == 0, fill
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [1, 0])
def test_both_sample_paths(R, spread):
    """Chunks of 1 (pixel-bound), 2 to 1985 (spread) and 1986 (over the 1 GiB finished-sample budget: pixel-bound)."""
    h, w = 4, 8
    split = [(0, 1), (1, 3), (3, 10), (10, 11), (11, 75), (75, 2060), (2060, 4046)]
    S = split[-1][1]
    ctx, pr = _ctx(R, "irreg", h, w, wq_spread=spread)
    want_pix, want_rgb = _one_shot(ctx, pr, h, w, S)
    colours = _gpu_colours(R, ctx, pr, h, w, S)
    acc, pix, rgb = _chain(ctx, pr, h, w, split)
    _check_against(acc, pix, rgb, sequential_sum(colours, 0, S), want_pix, want_rgb, f"wq_spread={spread}")
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS + [{"wq_packet": 24}, {"wq_packet": 0}], ids=str)
def test_every_plan(R, plan):
    h, w, S = 203, 301, 16
    split = [(0, 1), (1, 5), (5, 16)]
    ref, pr0 = _ctx(R, "irreg", h, w)
    want_pix, want_rgb = _one_shot(ref, pr0, h, w, S)
    want_acc = _chain(ref, pr0, h, w, [(0, S)])[0]
    ref.close()
    ctx, pr = _ctx(R, "irreg", h, w, **plan)
    acc, pix, rgb = _chain(ctx, pr, h, w, split)
    _check_against(acc, pix, rgb, want_acc, want_pix, want_rgb, str(plan))
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["rgbbox_x255", "irreg_x255", "rgbbox_top_down", "rgbbox_negative"])
def test_out_of_range_scenes(R, scene):
    h, w, S = 37, 53, 9
    ctx, pr = _ctx(R, scene, h, w)
    want_pix, want_rgb = _one_shot(ctx, pr, h, w, S)
    whole = _chain(ctx, pr, h, w, [(0, S)])
    for split in ([(0, 1), (1, 2), (2, 9)], [(0, 4), (4, 9)]):
        acc, pix, rgb = _chain(ctx, pr, h, w, split)
        _check_against(acc, pix, rgb, whole[0], want_pix, want_rgb, str(split))
    o_pix, o_rgb, _ = O.Scene.custom(*SCENES[scene]()).prepare(h, w).render(h, w, S, want_rgb=True)
    assert (whole[1] == o_pix).all() and bits_differ(whole[2], o_rgb) == 0, "oracle"
    ctx.close()


@pytest.mark.gpu
def test_golden_frames_through_one_call(R, golden):
    for name, (pixels, meta) in golden.items():
        h, w = meta["shape"]
        ctx, pr = _ctx(R, name.split("_")[0], h, w)
        _, pix, _ = _chain(ctx, pr, h, w, [(0, 1)])
        assert (pix == pixels).all(), name
        ctx.close()


@pytest.mark.gpu
def test_million_spheres(R):
    h = w = 512
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_random(1 << 20, 1))
        want_pix, want_rgb = _one_shot(ctx, pr, h, w, 16)
        acc, pix, rgb = _chain(ctx, pr, h, w, [(0, 4), (4, 8), (8, 12), (12, 16)])
        whole = _chain(ctx, pr, h, w, [(0, 16)])
        _check_against(acc, pix, rgb, whole[0], want_pix, want_rgb, "1 M spheres")


# ------------------------------------------------------------------------------------------ GPU: shards, streams, errors


def _owned(h, w, rank, world):
    tiles_x = (w + 7) // 8
    j, i = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return ((j // 4) * tiles_x + i // 8) % world == rank


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_shards_write_only_their_pixels(R, world):
    torch = _torch()
    h, w, split = 101, 203, [(0, 3), (3, 4), (4, 12)]
    ctx, pr = _ctx(R, "irreg", h, w)
    full = _chain(ctx, pr, h, w, split)
    union = [np.zeros((h, w, 3), np.float32), np.zeros((h, w), np.int32), np.zeros((h, w, 3), np.float32)]
    for rank in range(world):
        ctx.set_shard(rank, world)
        accum = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda")
        pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
        rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        for a, b in split:
            ctx.render_accumulate_into(accum.data_ptr(), h, w, pr, a, b, pix.data_ptr(), rgb.data_ptr())
        ctx.sync()
        mine = _owned(h, w, rank, world)
        got = [_np(accum), _np(pix), _np(rgb)]
        for k, g in enumerate(got):
            assert (g[~mine] == SENTINEL).all(), (rank, k, "wrote another rank's pixels")
            union[k][mine] = g.view(union[k].dtype)[mine]
    ctx.set_shard(0, 1)
    assert bits_differ(union[0], full[0]) == 0 and (union[1] == full[1]).all() and bits_differ(union[2], full[2]) == 0
    ctx.close()


@pytest.mark.gpu
def test_renders_around_accumulation_plan_and_launch_as_before(R):
    """A render's frame and launches do not depend on accumulation calls in between (learned order, heavy-first probe)."""
    torch = _torch()
    h, w = 250, 250
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")

    def run(with_accum):
        ctx, pr = _ctx(R, "irreg", h, w)
        accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        frames, launches = [], []
        for spp in (1, 1, 4, 1, 4):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            launches.append(ctx.launch_count() - n0)
            frames.append(_np(out))
            if with_accum:
                for a, b in ((0, 1), (1, 4), (4, 5)):
                    n0 = ctx.launch_count()
                    ctx.render_accumulate(pr, accum, a, b)
                    assert ctx.launch_count() - n0 == 1, "one launch per call"
        ctx.close()
        return frames, launches

    plain, accumulated = run(False), run(True)
    assert plain[1] == accumulated[1]
    assert plain[1][0] > 1 and plain[1][1] == 1, "the learned order is recorded by the first frame and used by the second"
    for a, b in zip(plain[0], accumulated[0]):
        assert (a == b).all()


@pytest.mark.gpu
def test_torch_stream_and_freeing_the_scene_in_flight(R):
    torch = _torch()
    h, w, S = 300, 400, 8
    ctx, pr = _ctx(R, "rgbbox", h, w)
    want_acc, want_pix, want_rgb = _chain(ctx, pr, h, w, [(0, S)])
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        acc, pix, rgb = _chain(ctx, pr, h, w, [(0, 2), (2, S)])
    _check_against(acc, pix, rgb, want_acc, want_pix, want_rgb, "torch stream")
    ctx.set_stream(None)
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for a, b in ((0, 3), (3, S)):
        s, c = SCENES["rgbbox"]()
        pr2 = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        ctx.render_accumulate_into(accum.data_ptr(), h, w, pr2, a, b, pix.data_ptr())
        pr2.free()          # while the call may still be in flight
    ctx.sync()
    assert bits_differ(_np(accum), want_acc) == 0 and (_np(pix) == want_pix).all()
    ctx.close()


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w = 37, 53
    ctx, pr = _ctx(R, "rgbbox", h, w)
    want = _chain(ctx, pr, h, w, [(0, 3)])
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    pix = torch.empty((h, w), dtype=torch.int32, device="cuda")

    class Freed:
        handle = None

    cases = [
        (dict(s_begin=-1, s_end=3), "bad sample range"),
        (dict(s_begin=3, s_end=3), "bad sample range"),
        (dict(s_begin=4, s_end=3), "bad sample range"),
        (dict(s_begin=-5, s_end=0), "bad sample range"),
        (dict(accum=None), "accum_dev is required"),
        (dict(h=0), "bad image size"),
        (dict(w=65537), "bad image size"),
        (dict(prepared=Freed()), "invalid prepared scene"),
    ]
    for change, message in cases:
        args = dict(accum=accum.data_ptr(), h=h, w=w, prepared=pr, s_begin=0, s_end=3)
        args.update(change)
        with pytest.raises(R.RayError, match=message):
            ctx.render_accumulate_into(args["accum"], args["h"], args["w"], args["prepared"], args["s_begin"], args["s_end"],
                                       pix.data_ptr())
        ctx.render_accumulate_into(accum.data_ptr(), h, w, pr, 0, 3, pix.data_ptr())
        ctx.sync()
        assert bits_differ(_np(accum), want[0]) == 0 and (_np(pix) == want[1]).all(), message
    good = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
    for bad in (good.cpu(), good.double(), good[:, :, :2], good.transpose(0, 1), good.reshape(h, w * 3), np.zeros((h, w, 3), np.float32)):
        with pytest.raises(ValueError):
            ctx.render_accumulate(pr, bad, 0, 1)
    ctx.close()


@pytest.mark.gpu
def test_largest_frame(R):
    """2^30 pixels: accum offsets pass 2^32 bytes (12 GiB of sums)."""
    torch = _torch()
    h = w = 32768
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.irreg())
        want = torch.empty((h, w), dtype=torch.int32, device="cuda")
        ctx.render_into(want.data_ptr(), h, w, pr, spp=2)
        pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        for a, b in ((0, 1), (1, 2)):
            ctx.render_accumulate_into(accum.data_ptr(), h, w, pr, a, b, pix.data_ptr())
        ctx.sync()
        assert torch.equal(pix, want)
        rows = [0, 1, h // 2, h - 1]
        chunked = accum[rows].cpu().numpy()
        ctx.render_accumulate_into(accum.data_ptr(), h, w, pr, 0, 2, None)
        ctx.sync()
        assert bits_differ(accum[rows].cpu().numpy(), chunked) == 0
        assert not np.isnan(chunked).any()
        del accum, pix, want
        torch.cuda.empty_cache()
