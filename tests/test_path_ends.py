"""The colour of a path that ends short of the sky: absorbed (scatter gives #none) or cut at the depth limit.

ray_colour (ray.fut:126-148) ends a path in one of three ways.  At the sky the colour is `light * sky`.  Absorbed, it is
`light * colour`; at the depth limit, after the last scatter, `light_old * colour`.  `colour` starts at +0 and is only
ever multiplied by the light, so at those two ends it is +0, -0 (an odd number of the lights it met had their sign bit
set) or NaN (a light overflowed to inf: inf * 0 = NaN), and a NaN channel quantises to INT32_MIN, not 0.  The built-in
scenes never show this: their colours are in [0, 1].  The scenes here do: the input-range scenes of
test_input_ranges.py, an rgbbox with a signed palette of colours, and a room (small spheres inside one enclosing sphere,
the camera inside it) where no path reaches the sky.

On the CPU, `ray_colour_f32` restates ray_colour in numpy float32 on top of a closest-hit query at (0, 1e9), with the
oracle's operation order, and reports each path's end.  It equals the oracle's trace_paths bit for bit, and every case
the GPU tests run has a floor of absorbed or depth-limited ends whose colour is -0.0 or NaN, so none passes by judging
nothing.  On the GPU: path queries, frames through every kernel and entry point, scene batches, progressive and
adaptive frames and every staging plan, bit for bit against the oracle (any NaN equals any NaN)."""
import functools

import numpy as np
import pytest

import ray_query_oracle as Q   # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ, quantise, random_rays
from test_input_ranges import KERNELS, PIXEL_SCENES
from test_render_accumulate import frame_of, sequential_sum
from test_render_adaptive_var import m2_model
from test_render_gbuffer import _gb_into, differ, oracle_gbuffer
from test_staging_plans import FORCED_PLANS, STAGING, expect, staging, variant

F = np.float32
SKY, ABSORBED, DEPTH_LIMIT = 1, 2, 3
PALETTE = np.float32([-1, -0.5, -0.0, 0.0, 0.5, 1, 255, -255, 1e30, -1e30])
DEPTHS = list(range(9)) + [50]
SMALL = (37, 53)     # partial tiles on both edges
LARGE = (500, 500)

# ------------------------------------------------------------------------------------------ scenes


def signed_palette():
    """rgbbox with every colour channel drawn from PALETTE"""
    s, c = O.Scene.named("rgbbox").arrays()
    s = s.copy()
    s[:, 3:6] = PALETTE[np.random.default_rng(11).integers(0, len(PALETTE), (len(s), 3))]
    return s, c


def room():
    """200 small spheres coloured from PALETTE inside one enclosing sphere (radius 60, centre 0), the camera inside it
    and outside every small sphere: no camera path reaches the sky, every one ends absorbed by the room's wall (its
    normal points out, so the reflection goes back in) or at the depth limit."""
    rng = np.random.default_rng(12)
    cam = np.float32([0, 0, 45, 0, 0, 0, 60])
    small = []
    while len(small) < 200:
        p = rng.uniform(-38, 38, 3)
        r = rng.uniform(1.5, 4.0)
        if np.linalg.norm(p) + r < 55 and np.linalg.norm(p - cam[:3]) > r + 2:
            small.append([*p, 0, 0, 0, r])
    s = np.float32(small + [[0, 0, 0, 0, 0, 0, 60]])
    s[:, 3:6] = PALETTE[rng.integers(0, len(PALETTE), (len(s), 3))]
    return s, cam


SCENES = {
    **{k: PIXEL_SCENES[k] for k in ("rgbbox_negative", "rgbbox_1e30_black", "rgbbox_x255", "irreg_x255")},
    "signed_palette": signed_palette,
    "room": room,
}
# the frame size each scene is rendered at
FRAME = {"rgbbox_negative": LARGE, "rgbbox_1e30_black": LARGE, "rgbbox_x255": LARGE, "irreg_x255": LARGE,
         "signed_palette": SMALL, "room": SMALL}
FRAME_SCENES = ["rgbbox_negative", "rgbbox_1e30_black", "rgbbox_x255", "irreg_x255", "room"]


@functools.lru_cache(maxsize=None)
def scene(name):
    s, c = SCENES[name]()
    s, c = np.ascontiguousarray(s, F), np.ascontiguousarray(c, F)
    s.setflags(write=False)
    c.setflags(write=False)
    return s, c


@functools.lru_cache(maxsize=None)
def query_oracle(name, h=SMALL[0], w=SMALL[1]):
    return Q.prepare_custom(*scene(name), h, w)


# ------------------------------------------------------------------------------------------ rays


def _unit(rng, n):
    d = rng.standard_normal((n, 3)).astype(F)
    return d / np.linalg.norm(d, axis=1, keepdims=True).astype(F)


def ray_sets(name, n=4000):
    """{kind: float32 [m, 6]}: random rays, the scene's frame's camera rays, rays from 0.05 outside a sphere's surface
    and rays from inside a sphere, all with unit directions except the camera rays"""
    import raytracers_b200 as R
    s, _ = scene(name)
    rng = np.random.default_rng(len(name))
    geo = s[np.isfinite(s).all(1)]
    pick = geo[rng.integers(0, len(geo), n)]
    u = _unit(rng, n)
    outside = np.concatenate([pick[:, :3] + u * (pick[:, 6:7] + F(0.05)), _unit(rng, n)], 1)
    inside = np.concatenate([pick[:, :3] + u * (pick[:, 6:7] * F(rng.uniform(0, 0.9, (n, 1)))), _unit(rng, n)], 1)
    cam = R.camera_rays(query_oracle(name, *FRAME[name]).camera(), *FRAME[name]).reshape(-1, 6)
    return {"random": random_rays(geo, n, len(name) + 1), "camera": cam,
            "outside": np.ascontiguousarray(outside, F), "inside": np.ascontiguousarray(inside, F)}


# ------------------------------------------------------------------------------------------ the restatement


def _dot(a, b):
    m = a * b
    return (m[..., 0] + m[..., 1]) + m[..., 2]          # prim.fut:22-24, left to right


def _normalise(v):
    return (F(1) / np.sqrt(_dot(v, v)))[..., None] * v  # prim.fut:26-28: scale (1 / norm v) v


def ray_colour_f32(closest_hits, colours, rays, max_depth):
    """ray_colour (ray.fut:126-148) in numpy float32 of every ray of float32 [n, 6], each segment's objs_hit from
    closest_hits(rays [m, 6]) -> float32 [m, 8] records (t, bits(sphere), p, normal) at (0, 1e9), colours float32
    [spheres, 3] the caller's sphere colours.  Returns (rgb float32 [n, 3], objs_hit calls int32 [n], end int8 [n]:
    0 = the loop never ran, SKY, ABSORBED or DEPTH_LIMIT)."""
    r = np.array(rays, F).reshape(-1, 6)
    n = len(r)
    light, colour = np.ones((n, 3), F), np.zeros((n, 3), F)
    segs, end = np.zeros(n, np.int32), np.zeros(n, np.int8)
    alive = np.full(n, max_depth > 0)
    with np.errstate(all="ignore"):
        for depth in range(max_depth):   # every live path has made `depth` scatters
            idx = np.nonzero(alive)[0]
            if len(idx) == 0:
                break
            segs[idx] += 1
            rec = np.asarray(closest_hits(r[idx]), F).reshape(-1, 8)
            sph = np.ascontiguousarray(rec[:, 1]).view(np.int32)
            hit = sph >= 0
            d, nrm = r[idx, 3:6], rec[:, 5:8]
            unit = _normalise(d)
            refl = unit - (F(2) * _dot(unit, nrm))[:, None] * nrm                 # reflect, ray.fut:116-117
            scat = hit & (_dot(refl, nrm) > F(0))                                # scatter, ray.fut:119-124
            t = F(0.5) * (unit[:, 1] + F(1))                                     # the sky, ray.fut:141-148
            sky = (F(1) - t)[:, None] * F(1) + t[:, None] * F([0.5, 0.7, 1.0])
            li, ci = light[idx], colour[idx]
            new_colour = np.where(~hit[:, None], li * sky, li * ci)
            ends = np.where(~hit, SKY, np.where(scat, DEPTH_LIMIT if depth + 1 == max_depth else 0, ABSORBED)).astype(np.int8)
            light[idx] = np.where(scat[:, None], li * colours[np.where(scat, sph, 0)], li)   # ray.fut:135
            colour[idx] = new_colour
            r[idx[scat], :3] = rec[scat, 2:5]
            r[idx[scat], 3:6] = refl[scat]
            end[idx] = ends
            alive[idx[ends != 0]] = False
    return colour, segs, end


def signed_ends(rgb, end):
    """Absorbed and depth-limited ends with a -0.0 or NaN channel: where a +0 end colour is wrong"""
    rgb = np.asarray(rgb, F)
    odd = (np.isnan(rgb) | ((rgb == 0) & np.signbit(rgb))).any(1)
    return int((odd & ((end == ABSORBED) | (end == DEPTH_LIMIT))).sum())


def assert_paths(got_rgb, got_seg, want_rgb, want_seg, what):
    bad = bits_differ(got_rgb, want_rgb)
    assert bad == 0, f"{what}: {bad} colour values differ"
    bad = int((np.asarray(got_seg).ravel() != np.asarray(want_seg).ravel()).sum())
    assert bad == 0, f"{what}: {bad} segment counts differ"


# The least number of absorbed and depth-limited ends whose colour is -0.0 or NaN: per scene over all its ray sets and
# DEPTHS (PATH_FLOOR), and among its frame's spp 1 camera rays (FRAME_FLOOR).  Well below what the cases have, except on
# the input-range scenes' frames: there only a few long paths of the 500 x 500 frame overflow or turn negative.
PATH_FLOOR = {"rgbbox_negative": 1000, "rgbbox_1e30_black": 500, "rgbbox_x255": 1, "irreg_x255": 1, "signed_palette": 1000,
              "room": 1000}
FRAME_FLOOR = {"rgbbox_negative": 1, "rgbbox_1e30_black": 1, "rgbbox_x255": 1, "irreg_x255": 1, "room": 100}


# ------------------------------------------------------------------------------------------ CPU


def test_room_premises():
    """No camera path of the room reaches the sky; the camera is outside every small sphere and inside the room."""
    s, c = scene("room")
    assert np.linalg.norm(s[:-1, :3] - c[:3], axis=1).min() > s[:-1, 6].max()
    o = query_oracle("room")
    rays = ray_sets("room")["camera"]
    for depth in (1, 3, 50):
        _, _, end = ray_colour_f32(o.trace_hits, s[:, 3:6], rays, depth)
        assert not (end == SKY).any(), depth


@pytest.mark.parametrize("name", list(SCENES))
def test_restatement_equals_the_oracle(name):
    """ray_colour_f32 on the oracle's closest hits is the oracle's trace_paths bit for bit, colours and segments, on
    every ray set at every depth the GPU tests use, with at least PATH_FLOOR ends that a +0 rule gets wrong."""
    s, _ = scene(name)
    o = query_oracle(name)
    found = 0
    for kind, rays in ray_sets(name).items():
        for depth in DEPTHS:
            rgb, seg, end = ray_colour_f32(o.trace_hits, s[:, 3:6], rays, depth)
            want_rgb, want_seg = o.trace_paths(rays, depth)
            assert_paths(rgb, seg, want_rgb, want_seg, f"{name} {kind} max_depth {depth}")
            if depth == 0:   # the loop never runs: +0
                assert (end == 0).all() and not np.signbit(rgb).any() and (rgb == 0).all()
            else:
                assert (end != 0).all()
            found += signed_ends(rgb, end)
    assert found >= PATH_FLOOR[name], f"{name}: {found} -0.0 / NaN ends"


@functools.lru_cache(maxsize=None)
def camera_colours(name, spp):
    """The oracle's colour of every sample's camera ray of the scene's frame: float32 [h, w, spp, 3]"""
    import raytracers_b200 as R
    h, w = FRAME[name]
    o = query_oracle(name, h, w)
    return o.trace_paths(R.camera_rays(o.camera(), h, w, spp).reshape(-1, 6))[0].reshape(h, w, spp, 3)


@functools.lru_cache(maxsize=None)
def oracle_frame(name, spp, cam7=None):
    """The oracle's (pixels [h][w], rgb [h][w][3]) of the scene's frame, with another camera where given"""
    s, c = scene(name)
    h, w = FRAME[name]
    pix, rgb, _ = O.Scene.custom(s, c if cam7 is None else np.float32(cam7)).prepare(h, w).render(h, w, spp, want_rgb=True)
    return pix, rgb


@pytest.mark.parametrize("name", FRAME_SCENES)
def test_frame_premises(name):
    """Each frame's spp 1 camera rays have their floor of -0.0 / NaN non-sky ends, the frame is the quantised colour of
    those rays, and a +0 at the non-sky ends (the rule the kernels once followed) changes packed pixels of the frame."""
    import raytracers_b200 as R
    s, _ = scene(name)
    h, w = FRAME[name]
    o = query_oracle(name, h, w)
    rays = R.camera_rays(o.camera(), h, w).reshape(-1, 6)
    rgb, _, end = ray_colour_f32(o.trace_hits, s[:, 3:6], rays, 50)
    assert signed_ends(rgb, end) >= FRAME_FLOOR[name], name
    pix, want_rgb = oracle_frame(name, 1)
    assert bits_differ(rgb.reshape(h, w, 3), want_rgb) == 0
    assert (quantise(rgb.reshape(h, w, 3)) == pix).all()
    plus = np.where(((end == ABSORBED) | (end == DEPTH_LIMIT))[:, None], F(0), rgb)
    assert int((quantise(plus) != quantise(rgb)).sum()) > 0, name


# ------------------------------------------------------------------------------------------ GPU helpers


def _gpu_hits(ctx, pr):
    """closest_hits for ray_colour_f32 through the library's own trace_hits at (0, 1e9)"""
    def hits(rays):
        if len(rays) == 0:
            return np.zeros((0, 8), F)
        out = ctx.trace_hits(pr, _dev(rays), t_min=0.0, t_max=1e9)
        return np.concatenate([_np(out["t"])[:, None], _np(out["sphere"]).view(F)[:, None], _np(out["p"]),
                               _np(out["normal"])], 1)
    return hits


def _prepare(ctx, name, h=None, w=None):
    s, c = scene(name)
    fh, fw = FRAME[name]
    return ctx.prepare_scene(h or fh, w or fw, ctx.scene_from_arrays(s, c))


def _frame_into(ctx, pr, h, w, spp):
    torch = _torch()
    pix = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb)


def assert_frame(pix, rgb, want, what):
    bad = int((np.asarray(pix) != want[0]).sum())
    assert bad == 0, f"{what}: {bad} of {want[0].size} pixels differ from the oracle"
    if rgb is not None:
        bad = bits_differ(rgb, want[1])
        assert bad == 0, f"{what}: {bad} float framebuffer values differ from the oracle"


# ------------------------------------------------------------------------------------------ GPU: path queries


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_trace_paths_equals_the_oracle(R, name):
    """trace_paths at max_depth 0-8 and 50 on random, camera, just-outside and inside rays: colours and segments bit
    for bit the oracle's; and the restatement driven by the library's own trace_hits is its trace_paths."""
    s, c = scene(name)
    o = query_oracle(name)
    with R.Context() as ctx:
        pr = ctx.prepare_scene(*SMALL, ctx.scene_from_arrays(s, c))
        hits = _gpu_hits(ctx, pr)
        for kind, rays in ray_sets(name).items():
            d = _dev(rays)
            for depth in DEPTHS:
                rgb, seg = ctx.trace_paths(pr, d, max_depth=depth)
                rgb, seg = _np(rgb), _np(seg)
                what = f"{name} {kind} max_depth {depth}"
                assert_paths(rgb, seg, *o.trace_paths(rays, depth), what + " vs the oracle")
                if depth in (1, 2, 3, 8):
                    mine, my_seg, _ = ray_colour_f32(hits, s[:, 3:6], rays, depth)
                    assert_paths(rgb, seg, mine, my_seg, what + " vs the restatement on the library's trace_hits")


@pytest.mark.gpu
def test_scene_batch_paths_equal_the_oracle(R):
    """trace_scene_batch_paths on a batch of the 400-sphere scenes here (and rgbbox): every member's colours and
    segments bit for bit the oracle's, at every depth."""
    names = ["rgbbox_negative", "rgbbox_1e30_black", "rgbbox_x255", "signed_palette"]
    s = np.stack([scene(k)[0] for k in names] + [O.Scene.named("rgbbox").arrays()[0]])
    cams = np.stack([scene(k)[1] for k in names] + [O.Scene.named("rgbbox").arrays()[1]])
    rays = np.stack([ray_sets(k, 1000)[kind][:1000] for k in names for kind in ("random",)]
                    + [random_rays(s[-1], 1000, 3)])
    oracles = [Q.prepare_custom(s[b], cams[b], *SMALL) for b in range(len(s))]
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(*SMALL, _dev(s), cams)
        d = _dev(rays)
        for depth in DEPTHS:
            rgb, seg = ctx.trace_scene_batch_paths(batch, d, max_depth=depth)
            rgb, seg = _np(rgb), _np(seg)
            for b in range(len(s)):
                assert_paths(rgb[b], seg[b], *oracles[b].trace_paths(rays[b], depth), f"member {b} max_depth {depth}")


# ------------------------------------------------------------------------------------------ GPU: frames


def _kernel_runs():
    return [(k, {}) for k in KERNELS if k != "warpqueue"] + [("warpqueue", {"wq_spread": 0}), ("warpqueue", {"wq_spread": 1})]


@pytest.mark.gpu
@pytest.mark.parametrize("name", FRAME_SCENES)
def test_frames_every_kernel(R, name):
    """render_host at spp 1, 3 and 16 through every kernel: packed pixels and the float framebuffer are the oracle's"""
    h, w = FRAME[name]
    for kernel, tuning in _kernel_runs():
        with R.Context(kernel=kernel, **tuning) as ctx:
            pr = _prepare(ctx, name)
            for spp in (1, 3, 16):
                pix, rgb = ctx.render_host(h, w, pr, spp=spp, want_rgb=True)
                assert_frame(pix, rgb, oracle_frame(name, spp), f"{name} {kernel} {tuning} spp {spp}")


def _second_camera(name):
    c = np.array(scene(name)[1])
    c[0:3] = c[0:3] * F(0.8) + F([3, -2, 1])
    return tuple(float(x) for x in c)


@pytest.mark.gpu
@pytest.mark.parametrize("name", FRAME_SCENES)
def test_frames_every_entry_point(R, name):
    """The same frames through render_into, render_batch, shards de-tiled at world 2 and 3, views, a device-prepared
    scene and a scene batch"""
    torch = _torch()
    from raytracers_b200 import distributed as D
    s, c = scene(name)
    h, w = FRAME[name]
    want = {spp: oracle_frame(name, spp) for spp in (1, 3, 16)}
    with R.Context() as ctx:
        ctx.set_stream(torch.cuda.current_stream().cuda_stream)
        pr = _prepare(ctx, name)
        for spp in (1, 3, 16):
            assert_frame(*_frame_into(ctx, pr, h, w, spp), want[spp], f"{name} render_into spp {spp}")
        jobs = [(1, True), (16, True), (3, False)]
        pix = [torch.full((h, w), -1, dtype=torch.int32, device="cuda") for _ in jobs]
        rgb = [torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda") for _ in jobs]
        ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=spp, out_dev=p.data_ptr(), out_rgb_dev=q.data_ptr() if with_rgb else None)
                          for (spp, with_rgb), p, q in zip(jobs, pix, rgb)])
        torch.cuda.synchronize()
        for (spp, with_rgb), p, q in zip(jobs, pix, rgb):
            assert_frame(_np(p), _np(q) if with_rgb else None, want[spp], f"{name} render_batch spp {spp}")
        for world in (2, 3):
            padded = D.tile_layout(h, w, world)[3]
            gathered = torch.full((world, padded, 32), -1, dtype=torch.int32, device="cuda")
            for rank in range(world):
                ctx.set_shard(rank, world)
                ctx.render_shard_into(gathered[rank].data_ptr(), h, w, pr, spp=3)
                torch.cuda.synchronize()
            ctx.set_shard(0, 1)
            frame = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
            ctx.detile(gathered.data_ptr(), frame.data_ptr(), h, w, world)
            torch.cuda.synchronize()
            assert_frame(_np(frame), None, want[3], f"{name} shards world {world}")
        cam2 = _second_camera(name)
        cams = np.stack([c, np.float32(cam2)])
        for spp in (1, 3):
            vp, vr = ctx.render_views(pr, cams, h, w, spp, want_rgb=True)
            assert_frame(_np(vp[0]), _np(vr[0]), want[spp], f"{name} view 0 spp {spp}")
            assert_frame(_np(vp[1]), _np(vr[1]), oracle_frame(name, spp, cam2), f"{name} view 1 spp {spp}")
        dev = ctx.prepare_scene_device(h, w, _dev(s), c)
        for spp in (1, 16):
            assert_frame(*_frame_into(ctx, dev, h, w, spp), want[spp], f"{name} device-prepared spp {spp}")
        batch = ctx.prepare_scene_batch(h, w, _dev(np.stack([s, s])), np.stack([c, np.float32(cam2)]))
        for spp in (1, 3):
            bp, br = ctx.render_scene_batch(batch, h, w, spp, want_rgb=True)
            assert_frame(_np(bp[0]), _np(br[0]), want[spp], f"{name} scene batch member 0 spp {spp}")
            assert_frame(_np(bp[1]), _np(br[1]), oracle_frame(name, spp, cam2), f"{name} scene batch member 1 spp {spp}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", FRAME_SCENES)
def test_progressive_and_adaptive_frames(R, name):
    """Progressive chains split at s_begin > 0 (where -0 + -0 stays -0 and NaN stays NaN), and adaptive chains with and
    without the variance: sums, M2, counts, pixels and floats against the oracle's per-sample colours"""
    torch = _torch()
    h, w = FRAME[name]
    colours = camera_colours(name, 16)
    with R.Context() as ctx:
        pr = _prepare(ctx, name)
        for split in ([(0, 1), (1, 3)], [(0, 5), (5, 16)], [(0, 1), (1, 2), (2, 16)]):
            accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
            for a, b in split:
                pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
                want_acc = sequential_sum(colours, 0, b)
                assert bits_differ(_np(accum), want_acc) == 0, f"{name} accumulate [{a}, {b}) sums"
                assert_frame(_np(pix), _np(rgb), frame_of(want_acc, b), f"{name} accumulate [{a}, {b})")
            assert_frame(_np(pix), _np(rgb), oracle_frame(name, split[-1][1]), f"{name} accumulate {split}")
        mask = np.random.default_rng(5).random((h, w)) < 0.5
        masks, n_adds = [None, mask, None], [1, 2, 13]
        want_acc, want_m2, want_cnt = m2_model(colours, masks, n_adds)
        for with_m2 in (False, True):
            accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
            m2 = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda") if with_m2 else None
            counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            pix = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
            rgb = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
            for m, n in zip(masks, n_adds):
                ctx.render_adaptive(pr, accum, counts, n, mask=None if m is None else torch.from_numpy(m).cuda(),
                                    pixels=pix, rgb=rgb, m2=m2)
                assert ctx.last_plan()["query"] == ("adaptive_var" if with_m2 else "adaptive")
            what = f"{name} adaptive{' with variance' if with_m2 else ''}"
            assert (_np(counts) == want_cnt).all(), f"{what}: counts"
            assert bits_differ(_np(accum), want_acc) == 0, f"{what}: sums"
            if with_m2:
                assert bits_differ(_np(m2), want_m2) == 0, f"{what}: M2"
            with np.errstate(all="ignore"):
                want_rgb = (F(1) / want_cnt.astype(F))[..., None] * want_acc
            assert_frame(_np(pix), _np(rgb), (quantise(want_rgb), want_rgb), what)


# ------------------------------------------------------------------------------------------ GPU: staging plans


@pytest.mark.gpu
def test_every_staging_plan_on_the_room(R):
    """The room's frames, progressive chunks, views and path queries through every staging case, K = 1 / 2, spread
    samples or not and the packet walk: every pixel instantiation and the path query's, against the oracle"""
    torch = _torch()
    s, c = scene("room")
    n = len(s)
    ni = n - 1
    h, w = SMALL
    caps = [("cap 0", 0, 4, 0), ("last node unstaged", 64 * (ni - 1), ni - 1, 0), ("nodes only", 64 * ni, ni, 0),
            ("one sphere short", 64 * ni + 16 * n - 16, ni, 0), ("whole", 64 * ni + 16 * n, ni, n), ("no cap", -1, ni, n)]
    cam2 = _second_camera("room")
    cams = np.stack([c, np.float32(cam2)])
    o = query_oracle("room")
    rays = np.concatenate([ray_sets("room", 1000)[k] for k in ("random", "outside", "inside")])
    want_paths = {depth: o.trace_paths(rays, depth) for depth in (3, 50)}
    colours = camera_colours("room", 3)
    launched, path_plans = set(), set()
    for cap_name, cap, nodes, spheres in caps:
        for plan in FORCED_PLANS:
            for packet in (0, 8):
                for spread in (1, 0):
                    what = f"room, {cap_name} (stage_cap {cap}), {plan}, wq_packet {packet}, wq_spread {spread}"
                    want = dict(kernel=R.KERNELS["warpqueue"], k=plan["wq_k"], warps=plan["wq_warps"], packet=packet,
                                smem_nodes=nodes, smem_spheres=spheres)
                    with R.Context(device=0, stage_cap=cap, wq_packet=packet, wq_spread=spread, **plan) as ctx:
                        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
                        for spp in ((1, 3) if spread else (3,)):
                            pix, rgb = _frame_into(ctx, pr, h, w, spp)
                            p = ctx.last_plan()
                            expect(p, f"{what}, spp {spp}", query="pixels", spread=int(spread and spp > 1), **want)
                            assert_frame(pix, rgb, oracle_frame("room", spp), f"{what}, spp {spp}")
                            launched.add(variant(p))
                        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
                        for a, b in ((0, 2), (2, 3)):
                            pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
                            p = ctx.last_plan()
                            expect(p, f"{what}, chunk [{a}, {b})", query="accumulate", spread=int(spread and b - a > 1), **want)
                            want_acc = sequential_sum(colours, 0, b)
                            assert bits_differ(_np(accum), want_acc) == 0, f"{what}, chunk [{a}, {b}): sums"
                            assert_frame(_np(pix), _np(rgb), frame_of(want_acc, b), f"{what}, chunk [{a}, {b})")
                            launched.add(variant(p))
                        for spp in ((1, 3) if spread else (3,)):
                            vp, vr = ctx.render_views(pr, cams, h, w, spp, want_rgb=True)
                            p = ctx.last_plan()
                            expect(p, f"{what}, views at spp {spp}", query="views", spread=int(spread and spp > 1), **want)
                            assert_frame(_np(vp[0]), _np(vr[0]), oracle_frame("room", spp), f"{what}, view 0 at spp {spp}")
                            assert_frame(_np(vp[1]), _np(vr[1]), oracle_frame("room", spp, cam2), f"{what}, view 1 at spp {spp}")
                            launched.add(variant(p))
                        if packet == 0 and spread == 1:
                            d = _dev(rays)
                            for depth, (want_rgb, want_seg) in want_paths.items():
                                rgb, seg = ctx.trace_paths(pr, d, max_depth=depth)
                                p = ctx.last_plan()
                                expect(p, f"{what}, paths", query="closest", ranged=0, **{k: v for k, v in want.items() if k != "packet"})
                                assert_paths(_np(rgb), _np(seg), want_rgb, want_seg, f"{what}, paths max_depth {depth}")
                                path_plans.add((p["k"], staging(p)))
    want_pixel = {(q, False, k, sp, pk, st) for q in ("pixels", "accumulate", "views") for k in (1, 2) for sp in (False, True)
                  for pk in (False, True) for st in STAGING.values()}
    assert launched == want_pixel, f"pixel instantiations not launched: {sorted(want_pixel - launched)}"
    assert path_plans == {(k, st) for k in (1, 2) for st in STAGING.values()}


# ------------------------------------------------------------------------------------------ GPU: G-buffer


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 3])
def test_gbuffer_of_the_room(R, spp):
    """First-hit buffers do not see path ends: the room's five buffers are the rule over the oracle's first hits"""
    s, c = scene("room")
    h, w = SMALL
    want = oracle_gbuffer(query_oracle("room"), s[:, 3:6], h, w, spp)
    assert (want["coverage"] == spp).all(), "every camera ray of the room hits a sphere"
    with R.Context() as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        differ(_gb_into(ctx, pr, h, w, spp), want, f"room gbuffer spp {spp}")
