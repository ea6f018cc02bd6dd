"""Scene inputs outside the ranges of the built-in scenes, which ray_b200_scene_from_arrays accepts as they are: colours
far above 1 or below 0, colours whose products overflow to inf and meet black spheres (NaN light), cameras that look
along vup or at their own position (a NaN camera basis, so NaN rays), scenes placed 2^20 and 2^30 times further out,
zero and negative radii, mixed signed zeros, and scenes so small that the intersection arithmetic runs on subnormal
numbers.

The CPU oracle is the judge everywhere.  Packed pixels follow one rule on both sides (include/ray_b200.h): each channel
is 255.99 * c truncated, or INT32_MIN where that is NaN or outside [-2^31, 2^31), packed with wrapping shifts
(`quantise`).  Float outputs are compared bit for bit, except that any NaN equals any NaN (`bits_differ`): a NaN's
bit pattern is not part of the contract."""
import functools

import numpy as np
import pytest

import ray_query_oracle as Q   # tests/ray_query_oracle.py: the CPU oracle of the per-call and the ranged ray queries
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ, hits_differ, quantise, random_rays

KERNELS = ["mega", "persistent", "wavefront", "warpqueue", "streamqueue", "lanewalk"]
H, W = 37, 53        # partial tiles on both edges
F32_TINY = np.float32(2.0 ** -126)   # the smallest normal float32

# ------------------------------------------------------------------------------------------ scenes


@functools.lru_cache(maxsize=None)
def _builtin(name):
    s, c = O.Scene.named(name).arrays()
    s.setflags(write=False)
    c.setflags(write=False)
    return s, c


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


def _scaled(name, e):
    """Sphere centres, radii and the camera times 2^e (exact in float32); the frame's shape is unchanged."""
    s, c = _builtin(name)
    f = np.float32(2.0 ** e)
    s, c = s.copy(), c.copy()
    s[:, [0, 1, 2, 6]] *= f
    c[:6] *= f
    return s, c


def _bright_and_black():
    """Colours 1e30, every third sphere black: a path's light overflows to inf and then meets a 0 (inf * 0 = NaN)."""
    s, c = _recolour("rgbbox", lambda col: np.full_like(col, 1e30))
    s[::3, 3:6] = 0
    return s, c


PIXEL_SCENES = {
    "rgbbox_x255": lambda: _recolour("rgbbox", lambda col: col * np.float32(255)),    # the 0-255 colour convention
    "irreg_x255": lambda: _recolour("irreg", lambda col: col * np.float32(255)),
    "rgbbox_1e30_black": _bright_and_black,
    "rgbbox_negative": lambda: _recolour("rgbbox", lambda col: col * np.float32(-255)),
    "rgbbox_x2": lambda: _recolour("rgbbox", lambda col: col * np.float32(2)),
    "rgbbox_top_down": lambda: _camera("rgbbox", (0, 40, 0), (0, 0, 0)),      # look_at - look_from parallel to vup
    "irreg_top_down": lambda: _camera("irreg", (0, 40, 0), (0, 0, 0)),
    "rgbbox_look_at_self": lambda: _camera("rgbbox", (0, 30, 30), (0, 30, 30)),
    "rgbbox_scaled_2^20": lambda: _scaled("rgbbox", 20),
    "irreg_scaled_2^20": lambda: _scaled("irreg", 20),
    "rgbbox_scaled_2^30": lambda: _scaled("rgbbox", 30),
    "irreg_scaled_2^30": lambda: _scaled("irreg", 30),
}
NAN_CAMERA = ("rgbbox_top_down", "irreg_top_down", "rgbbox_look_at_self")


def _zero_radii():
    """rgbbox with every other radius 0: boxes of zero extent and, where rounding makes the discriminant positive,
    hits whose normal (p - centre) / 0 is inf or NaN."""
    s, c = _builtin("rgbbox")
    s = s.copy()
    s[::2, 6] = 0
    return s, c


def _negative_radii():
    """rgbbox with every other radius negated: inverted leaf boxes and inner boxes folded from them."""
    s, c = _builtin("rgbbox")
    s = s.copy()
    s[1::2, 6] *= -1
    return s, c


def _signed_zeros():
    """Spheres on and around the axes whose centre coordinates are -0.0 or +0.0, with radii +0.0, -0.0 or 0.25: leaf
    boxes whose bounds are zeros of either sign, so every min / max fold over them meets -0.0 against +0.0."""
    rng = np.random.default_rng(20)
    n = 300
    s = np.zeros((n, 7), np.float32)
    zero = np.where(rng.random((n, 3)) < 0.5, np.float32(-0.0), np.float32(0.0))
    off = rng.uniform(-8, 8, (n, 3)).astype(np.float32)
    s[:, :3] = np.where(rng.random((n, 3)) < 0.7, zero, off)
    s[:, 3:6] = rng.uniform(0.2, 1, (n, 3))
    s[:, 6] = np.float32([0.0, -0.0, 0.25])[rng.integers(0, 3, n)]
    return s, np.float32([3, 4, 20, 0, 0, 0, 60])


GEOMETRY_SCENES = {
    "zero_radii": _zero_radii,
    "negative_radii": _negative_radii,
    "signed_zeros": _signed_zeros,
    "rgbbox_scaled_2^20": lambda: _scaled("rgbbox", 20),
    "rgbbox_scaled_2^30": lambda: _scaled("rgbbox", 30),
}


ALL_SCENES = {**PIXEL_SCENES, **GEOMETRY_SCENES}


def frame_size(scene):
    """H x W, except for the scaled scenes: at 48 x 64 some of their camera rays have a direction that cancels to 0
    (NaN pixels), at H x W none has."""
    return (48, 64) if "scaled" in scene else (H, W)


def scene_arrays(scene):
    return ALL_SCENES[scene]()


@functools.lru_cache(maxsize=None)
def oracle_frame(scene, spp):
    """The oracle's (pixels [h][w], rgb [h][w][3], work counters) of a PIXEL_SCENES / GEOMETRY_SCENES scene."""
    s, c = scene_arrays(scene)
    h, w = frame_size(scene)
    return O.Scene.custom(s, c).prepare(h, w).render(h, w, spp=spp, want_rgb=True)


def saturating(rgb):
    """A conversion that saturates and maps NaN to 0 (CUDA's cvt.rzi.s32.f32), packed like `quantise`: the rule the
    scenes below must tell apart from the oracle's."""
    with np.errstate(over="ignore", invalid="ignore"):
        v = (np.float32(255.99) * np.asarray(rgb, np.float32)).astype(np.float64)
    q = np.where(np.isnan(v), 0, np.clip(np.trunc(np.nan_to_num(v)), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
    q = (q & 0xffffffff).astype(np.uint32)
    return ((q[..., 0] << np.uint32(16)) | (q[..., 1] << np.uint32(8)) | q[..., 2]).view(np.int32)


def assert_frame(pix, rgb, want_pix, want_rgb, what):
    bad = int((np.asarray(pix) != want_pix).sum())
    assert bad == 0, f"{what}: {bad} of {want_pix.size} pixels differ from the oracle"
    if rgb is not None:
        assert bits_differ(rgb, want_rgb) == 0, f"{what}: float framebuffer differs from the oracle"


# ------------------------------------------------------------------------------------------ CPU: the rule and the scenes


@pytest.mark.parametrize("spp", [1, 3])
@pytest.mark.parametrize("scene", list(ALL_SCENES))
def test_oracle_pixels_follow_the_quantisation_rule(scene, spp):
    """The oracle's packed pixels are `quantise` of its own float framebuffer: this pins the rule, not the compiler."""
    pix, rgb, _ = oracle_frame(scene, spp)
    assert int((quantise(rgb) != pix).sum()) == 0


def _channels(scene):
    _, rgb, _ = oracle_frame(scene, 1)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.float32(255.99) * rgb


def test_scene_premises():
    """Each scene produces what it is there for, and the scenes that must tell the rule from a saturating conversion
    do: there the saturating model disagrees with the oracle."""
    big = np.float32(2.0 ** 31)
    for scene in ("rgbbox_x255", "irreg_x255"):
        v = _channels(scene)
        assert (np.isfinite(v) & (v >= big)).any(), scene
    scaled = tuple(k for k in PIXEL_SCENES if "scaled" in k)
    for scene in ("rgbbox_1e30_black",) + scaled:
        assert np.isnan(_channels(scene)).any(), scene
        assert not np.isnan(_channels(scene)).all(), scene
    v = _channels("rgbbox_negative")
    assert (v < 0).any() and (v > -big).any() and (v < -big).any()
    v = _channels("rgbbox_x2")
    assert (v >= 256).any() and np.isfinite(v).all() and (np.abs(v) < big).all()
    for scene in NAN_CAMERA:
        s, c = scene_arrays(scene)
        assert np.isnan(O.Scene.custom(s, c).prepare(H, W).dump()["cam"][3:]).all(), scene
        assert np.isnan(_channels(scene)).all(), scene
    for scene in ("rgbbox_x255", "irreg_x255", "rgbbox_1e30_black", "rgbbox_negative") + scaled + NAN_CAMERA:
        pix, rgb, _ = oracle_frame(scene, 1)
        assert int((saturating(rgb) != pix).sum()) > 0, scene
    for scene in ("rgbbox_x2",):
        pix, rgb, _ = oracle_frame(scene, 1)
        assert int((saturating(rgb) != pix).sum()) == 0, scene


def test_quantise_rule_known_answers():
    """The rule on single channels: truncation toward 0, INT32_MIN outside [-2^31, 2^31) and for NaN, wrapping shifts."""
    def px(r, g, b):
        return int(quantise(np.float32([[r, g, b]]) / np.float32(255.99))[0]) & 0xffffffff
    assert px(1, 2, 3) == 0x010203
    assert px(255.5, 0, 0) == 0xff0000
    assert px(0, 0, -1.5) == 0xffffffff                      # -1, packed with wrapping shifts
    assert px(0, 0, np.nan) == 0x80000000
    assert px(0, 0, 2.0 ** 31) == 0x80000000
    assert px(0, 0, 2.0 ** 31 - 128) == 0x7fffff80          # the largest float32 below 2^31
    assert px(0, 0, -2.0 ** 31) == 0x80000000                # in range
    assert px(0, 0, np.inf) == px(0, 0, -np.inf) == 0x80000000
    assert px(np.nan, np.nan, 0) == 0                        # INT32_MIN << 16 and << 8 wrap to 0


@pytest.mark.parametrize("scene", list(GEOMETRY_SCENES))
def test_host_lbvh_equals_the_oracle(R, scene):
    """The host builder (scene_host.cpp) on the geometry scenes: every array bit for bit, boxes including zero signs."""
    s, c = GEOMETRY_SCENES[scene]()
    want = O.Scene.custom(s, c).prepare(H, W).dump()
    got = R.host_lbvh(s)
    for k in ("morton", "perm", "left", "right", "parent"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    np.testing.assert_array_equal(got["boxes"].view(np.uint32), want["boxes"].view(np.uint32))


def test_signed_zero_scene_premise():
    """The signed-zero scene's leaf boxes have bounds -0.0 and +0.0 on the same axis, and its inner boxes keep zeros."""
    s, c = _signed_zeros()
    lo, hi = s[:, :3] - s[:, 6:7], s[:, :3] + s[:, 6:7]
    neg = lambda a: (a == 0) & np.signbit(a)   # noqa: E731
    pos = lambda a: (a == 0) & ~np.signbit(a)  # noqa: E731
    for a in (lo, hi):
        assert all(neg(a[:, k]).any() and pos(a[:, k]).any() for k in range(3))
    boxes = O.Scene.custom(s, c).prepare(H, W).dump()["boxes"]
    assert (boxes == 0).any()


# ------------------------------------------------------------------------------------------ subnormal intermediates

SUBNORMAL_SCALES = [62, 68, 74]


def _tiny_scene(e):
    """rgbbox with centres and radii times 2^-e: its (ray, sphere) discriminants are subnormal while roots exist."""
    return _scaled("rgbbox", -e)


def _tiny_rays(spheres, n=4000, seed=68):
    """Origins in and around the scene's bounding box, unit directions (random_rays)."""
    return random_rays(spheres, n, seed)


def _discriminants(spheres, rays):
    """sphere_t's discriminant (ray.fut:32-51, device_math.cuh) of every (ray, sphere) pair in float32, same order."""
    s = np.asarray(spheres, np.float32)
    r = np.asarray(rays, np.float32)
    oc = r[:, None, :3] - s[None, :, :3]
    d = r[:, None, 3:6]
    a = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    b = (oc[..., 0] * d[..., 0] + oc[..., 1] * d[..., 1]) + oc[..., 2] * d[..., 2]
    c = ((oc[..., 0] * oc[..., 0] + oc[..., 1] * oc[..., 1]) + oc[..., 2] * oc[..., 2]) - s[None, :, 6] * s[None, :, 6]
    return b * b - a * c


@pytest.mark.parametrize("e", SUBNORMAL_SCALES)
def test_subnormal_premise(e):
    """The oracle finds hits with t_min = 0, and some (ray, sphere) pairs have a positive subnormal discriminant: a build
    that flushed subnormals to zero would turn those into misses."""
    s, c = _tiny_scene(e)
    rays = _tiny_rays(s)
    disc = _discriminants(s, rays)
    assert ((disc > 0) & (disc < F32_TINY)).any()
    o = Q.prepare_custom(s, c, H, W)
    assert o.trace_occluded(rays, 0.0, 1e9).any()
    _, counts = o.trace_multi_hits(rays, 8, 0.0, 1e9)
    assert counts.sum() > 0


# ------------------------------------------------------------------------------------------ GPU: renders


def _render_runs(kernel):
    """(spp, tuning) of every render run on `kernel`: 1 spp, and 3 spp with the warp-queue kernel's samples spread over
    lanes and kept on one lane."""
    if kernel == "warpqueue":
        return [(1, {}), (3, {"wq_spread": 1}), (3, {"wq_spread": 0})]
    return [(1, {}), (3, {})]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("scene", list(ALL_SCENES))
def test_render_equals_oracle(R, scene, kernel):
    """Packed pixels equal the oracle's and the float framebuffer equals it (any NaN equal to any NaN)."""
    s, c = scene_arrays(scene)
    h, w = frame_size(scene)
    for spp, tuning in _render_runs(kernel):
        want_pix, want_rgb, _ = oracle_frame(scene, spp)
        with R.Context(kernel=kernel, **tuning) as ctx:
            pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
            pix, rgb = ctx.render_host(h, w, pr, spp=spp, want_rgb=True)
        assert_frame(pix, rgb, want_pix, want_rgb, f"{scene} {kernel} spp={spp} {tuning}")


OUTPUT_PATH_SCENES = ["rgbbox_x255", "rgbbox_1e30_black", "rgbbox_negative", "rgbbox_top_down", "irreg_scaled_2^20"]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", OUTPUT_PATH_SCENES)
def test_every_output_path(R, scene):
    """The same frames through render_into, the reference's render entry and render_spp, the compact shard layout
    de-tiled at world 2 and 3, and render_batch with two frames in flight."""
    torch = _torch()
    from raytracers_b200 import distributed as D
    s, c = scene_arrays(scene)
    h, w = frame_size(scene)
    want = {spp: oracle_frame(scene, spp) for spp in (1, 3)}
    with R.Context() as ctx:
        ctx.set_stream(torch.cuda.current_stream().cuda_stream)
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        for spp in (1, 3):
            pix = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
            rgb = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
            ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
            torch.cuda.synchronize()
            assert_frame(_np(pix), _np(rgb), want[spp][0], want[spp][1], f"{scene} render_into spp={spp}")
            img = ctx.render(h, w, pr, spp=None if spp == 1 else spp)   # futhark_entry_render / ray_b200_entry_render_spp
            ctx.sync()
            assert_frame(img.values(), None, want[spp][0], None, f"{scene} entry render spp={spp}")
            img.free()
        for world in (2, 3):
            padded = D.tile_layout(h, w, world)[3]
            gathered = torch.full((world, padded, 32), -1, dtype=torch.int32, device="cuda")
            for rank in range(world):
                ctx.set_shard(rank, world)
                ctx.render_shard_into(gathered[rank].data_ptr(), h, w, pr, spp=3)
                torch.cuda.synchronize()
                np.testing.assert_array_equal(_np(gathered[rank]), D.extract_rank_tiles(want[3][0], rank, world))
            ctx.set_shard(0, 1)
            frame = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
            ctx.detile(gathered.data_ptr(), frame.data_ptr(), h, w, world)
            torch.cuda.synchronize()
            assert_frame(_np(frame), None, want[3][0], None, f"{scene} sharded world={world}")
        jobs = [(1, True), (3, True), (3, False), (1, False)]
        pix = [torch.full((h, w), -1, dtype=torch.int32, device="cuda") for _ in jobs]
        rgb = [torch.zeros((h, w, 3), dtype=torch.float32, device="cuda") for _ in jobs]
        ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=spp, out_dev=p.data_ptr(), out_rgb_dev=q.data_ptr() if with_rgb else None)
                          for (spp, with_rgb), p, q in zip(jobs, pix, rgb)])
        torch.cuda.synchronize()
        for (spp, with_rgb), p, q in zip(jobs, pix, rgb):
            assert_frame(_np(p), _np(q) if with_rgb else None, want[spp][0], want[spp][1], f"{scene} render_batch spp={spp}")


@pytest.mark.gpu
@pytest.mark.parametrize("scene", [k for k in PIXEL_SCENES if k not in NAN_CAMERA])
def test_trace_paths_of_camera_rays_quantise_to_the_frame(R, scene):
    """trace_paths of the frame's camera rays, quantised by the rule, equals the frame; its colours equal the oracle's
    float framebuffer.  (The NaN-camera scenes are left out: non-finite ray components are outside the query contract.)"""
    s, c = scene_arrays(scene)
    h, w = frame_size(scene)
    want_pix, want_rgb, _ = oracle_frame(scene, 1)
    with R.Context() as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        frame = ctx.render_host(h, w, pr)
        rays = R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6)
        rgb, _ = ctx.trace_paths(pr, _dev(rays))
    rgb = _np(rgb).reshape(h, w, 3)
    assert bits_differ(rgb, want_rgb) == 0
    assert int((quantise(rgb) != frame).sum()) == 0
    assert int((frame != want_pix).sum()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("scene", NAN_CAMERA)
def test_work_counters_on_nan_rays(R, scene):
    """NaN camera rays pass every box on both sides and meet every sphere: count_work equals the oracle's segments,
    box tests and leaf tests (box_hit's merged early-outs against the reference's per-axis ones, every slab NaN)."""
    s, c = scene_arrays(scene)
    h, w = frame_size(scene)
    with R.Context() as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        for spp in (1, 3):
            _, _, cnt = oracle_frame(scene, spp)
            got = ctx.count_work(h, w, pr, spp=spp)
            assert (got["segments"], got["box_tests"], got["leaf_tests"]) == (cnt["segments"], cnt["box_tests"], cnt["leaf_tests"])
            assert cnt["leaf_tests"] == cnt["segments"] * len(s)   # the whole tree, every time


# ------------------------------------------------------------------------------------------ GPU: geometry and queries


@pytest.mark.gpu
@pytest.mark.parametrize("scene", list(GEOMETRY_SCENES))
def test_device_lbvh_equals_the_oracle(R, scene):
    """The device builder (bvh_build.cu) and the host builder against the oracle, bit for bit, zero signs included."""
    s, c = GEOMETRY_SCENES[scene]()
    want = O.Scene.custom(s, c).prepare(H, W).dump()
    with R.Context() as ctx, R.Context(host_build=1) as ctx_h:
        for what, cx in (("device", ctx), ("host", ctx_h)):
            pr = cx.prepare_scene(H, W, cx.scene_from_arrays(s, c))
            got = pr.dump()
            for k in ("morton", "perm", "left", "right", "parent"):
                np.testing.assert_array_equal(got[k], want[k], err_msg=f"{what} {k}")
            np.testing.assert_array_equal(got["boxes"].view(np.uint32), want["boxes"].view(np.uint32), err_msg=f"{what} boxes")
            np.testing.assert_array_equal(pr.info()["root_box"].view(np.uint32), want["boxes"][0].view(np.uint32))
            assert bits_differ(pr.info()["camera"], want["cam"]) == 0, f"{what} camera"


def _query_rays(spheres, seed):
    """Random rays (unit directions, origins in and around the scene) and rays aimed at sphere centres with unit
    directions: against a zero radius their discriminant is 0 up to rounding, so some of them hit."""
    s = np.asarray(spheres, np.float32)
    rays = random_rays(s, 2048, seed)
    rng = np.random.default_rng(seed + 1)
    aim = rays[:512].copy()
    d = s[rng.integers(0, len(s), 512), :3] - aim[:, :3]
    aim[:, 3:6] = d / np.linalg.norm(d, axis=1, keepdims=True).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([rays, aim]), np.float32)


def test_zero_radius_premise():
    """Rays aimed at zero-radius spheres hit some of them, with a normal (p - centre) / 0 that is not finite."""
    s, c = _zero_radii()
    o = Q.prepare_custom(s, c, H, W)
    hits = o.trace_hits(_query_rays(s, 7), 0.0, 1e38)
    hit = hits[:, 1].view(np.int32) >= 0
    assert (~np.isfinite(hits[hit][:, 5:8])).any()


def _per_ray_intervals(spheres, n, seed):
    s = np.asarray(spheres, np.float32)
    diag = float(np.linalg.norm((s[:, :3] + np.abs(s[:, 6:7])).max(0) - (s[:, :3] - np.abs(s[:, 6:7])).min(0)))
    rng = np.random.default_rng(seed)
    lo = np.where(rng.random(n) < 0.3, 0.0, rng.uniform(0, 0.5 * diag, n)).astype(np.float32)
    return lo, (lo + rng.exponential(0.5 * diag, n)).astype(np.float32)


def _ranged(rays, lo, hi):
    r = np.asarray(rays, np.float32)
    return np.ascontiguousarray(np.concatenate([r[:, :3], lo[:, None], r[:, 3:], hi[:, None]], 1), np.float32)


def _hit_records(out):
    torch = _torch()
    return _np(torch.cat([out["t"][..., None], out["sphere"].view(torch.float32)[..., None], out["p"], out["normal"]], -1))


def check_queries(ctx, pr, spheres, cam, rays, intervals, ranged_rays, ks=(1, 8)):
    """trace_hits, trace_occluded and trace_multi_hits (each k of ks) per call on every interval and ranged on
    `ranged_rays`, against the oracles; records compared NaN-aware.  Returns the number of hits the oracle found."""
    o = Q.prepare_custom(spheres, cam, H, W)
    d, d8 = _dev(rays), _dev(ranged_rays)
    found = 0
    for t_min, t_max in intervals:
        what = f"({t_min}, {t_max})"
        want = o.trace_hits(rays, t_min, t_max)
        found += int((want[:, 1].view(np.int32) >= 0).sum())
        assert hits_differ(_hit_records(ctx.trace_hits(pr, d, t_min=t_min, t_max=t_max)), want) == 0, f"hits {what}"
        got = _np(ctx.trace_occluded(pr, d, t_min=t_min, t_max=t_max))
        assert int((got != o.trace_occluded(rays, t_min, t_max)).sum()) == 0, f"occluded {what}"
        for k in ks:
            out = ctx.trace_multi_hits(pr, d, k, t_min=t_min, t_max=t_max)
            want_m, want_n = o.trace_multi_hits(rays, k, t_min, t_max)
            assert hits_differ(_hit_records(out).reshape(-1, 8), want_m.reshape(-1, 8)) == 0, f"multi k={k} {what}"
            assert int((_np(out["count"]) != want_n).sum()) == 0, f"multi count k={k} {what}"
    assert hits_differ(_hit_records(ctx.trace_hits(pr, d8)), o.trace_hits_ranged(ranged_rays)) == 0, "hits ranged"
    assert int((_np(ctx.trace_occluded(pr, d8)) != o.trace_occluded_ranged(ranged_rays)).sum()) == 0, "occluded ranged"
    for k in ks:
        out = ctx.trace_multi_hits(pr, d8, k)
        want_m, want_n = o.trace_multi_hits_ranged(ranged_rays, k)
        assert hits_differ(_hit_records(out).reshape(-1, 8), want_m.reshape(-1, 8)) == 0, f"multi ranged k={k}"
        assert int((_np(out["count"]) != want_n).sum()) == 0, f"multi ranged count k={k}"
    return found


@pytest.mark.gpu
@pytest.mark.parametrize("scene", list(GEOMETRY_SCENES))
def test_ray_queries_on_geometry_scenes(R, scene):
    s, c = GEOMETRY_SCENES[scene]()
    rays = _query_rays(s, 7)
    lo, hi = _per_ray_intervals(s, len(rays), 8)
    with R.Context() as ctx:
        pr = ctx.prepare_scene(H, W, ctx.scene_from_arrays(s, c))
        found = check_queries(ctx, pr, s, c, rays, [(0.0, 1e38), (0.1, 1e9)], _ranged(rays, lo, hi))
    assert found > 0


@pytest.mark.gpu
@pytest.mark.parametrize("e", SUBNORMAL_SCALES)
def test_subnormal_queries(R, e):
    """Occlusion and multi-hit queries with t_min = 0 on a scene scaled by 2^-e, where the discriminants of the hits
    are subnormal (test_subnormal_premise): the library must not flush them to zero."""
    s, c = _tiny_scene(e)
    rays = _tiny_rays(s)
    o = Q.prepare_custom(s, c, H, W)
    _, hi = _per_ray_intervals(s, len(rays), e)
    rays8 = _ranged(rays, np.zeros(len(rays), np.float32), hi)
    with R.Context() as ctx:
        pr = ctx.prepare_scene(H, W, ctx.scene_from_arrays(s, c))
        d, d8 = _dev(rays), _dev(rays8)
        want = o.trace_occluded(rays, 0.0, 1e9)
        assert want.any()
        assert int((_np(ctx.trace_occluded(pr, d, t_min=0.0, t_max=1e9)) != want).sum()) == 0
        assert int((_np(ctx.trace_occluded(pr, d8)) != o.trace_occluded_ranged(rays8)).sum()) == 0
        for k in (1, 8):
            out = ctx.trace_multi_hits(pr, d, k, t_min=0.0, t_max=1e9)
            want_m, want_n = o.trace_multi_hits(rays, k, 0.0, 1e9)
            assert hits_differ(_hit_records(out).reshape(-1, 8), want_m.reshape(-1, 8)) == 0, f"multi k={k}"
            assert int((_np(out["count"]) != want_n).sum()) == 0, f"multi count k={k}"
            out = ctx.trace_multi_hits(pr, d8, k)
            want_m, want_n = o.trace_multi_hits_ranged(rays8, k)
            assert hits_differ(_hit_records(out).reshape(-1, 8), want_m.reshape(-1, 8)) == 0, f"multi ranged k={k}"
            assert int((_np(out["count"]) != want_n).sum()) == 0, f"multi ranged count k={k}"
