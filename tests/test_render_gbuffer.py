"""The first-hit buffers of a frame (include/ray_b200.h ray_b200_render_gbuffer): sphere id, depth, normal, albedo and
coverage of each pixel's camera rays, in one launch.  The rule is stated on the ray queries: H_s = trace_hits(r_s, 0, 1e9)
of sample s's camera ray r_s; id and depth are H_0's sphere and t, coverage counts the samples that hit, and normal and
albedo are in-order f32 means of H_s.normal and of the hit sphere's colour (the sky colour of trace_paths(r_s,
max_depth = 1) on a miss).

On the CPU the rule is restated in numpy over the CPU ray-query oracle and checked against the oracle's frames: where no
sample hits, albedo is the frame's float framebuffer bit for bit, and at one sample coverage is id >= 0.  On the GPU every
output equals the rule on the CPU oracle (small frames) or on the GPU's own trace_hits / trace_paths (large ones), bit for
bit and NaN-aware, on every plan, staging point and instantiation the kind can launch."""
import itertools

import numpy as np
import pytest

import limit_scenes as LS
import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from oracle import pyoracle as O
from ray_query_cases import PLANS, _dev, _np, _torch, bits_differ
from test_input_ranges import ALL_SCENES, frame_size
from test_render_accumulate import SCENES
from test_render_adaptive_var import _pixel_rays
from test_staging_plans import FORCED_PLANS, H, W, _camera_rays, dense_scene, expect, forced, variant  # noqa: F401 (forced: fixture)

OUTPUTS = ("id", "depth", "normal", "albedo", "coverage")
SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes


# ------------------------------------------------------------------------------------------ the rule in numpy


def gbuffer_rule(hits, sky, colours, spp):
    """hits float32 [n, spp, 8] (struct ray_b200_hit of every sample's camera ray), sky float32 [n, spp, 3]
    (trace_paths(max_depth = 1) of the same rays), colours float32 [spheres, 3] (the caller's sphere colours): the five
    buffers of the n pixels, as ray_b200_render_gbuffer states them."""
    hits = np.asarray(hits, np.float32).reshape(-1, spp, 8)
    sky = np.asarray(sky, np.float32).reshape(-1, spp, 3)
    colours = np.asarray(colours, np.float32).reshape(-1, 3)
    sphere = np.ascontiguousarray(hits[..., 1]).view(np.int32)
    hit = sphere >= 0
    albedo_x = np.where(hit[..., None], colours[np.where(hit, sphere, 0)], sky)
    normal_x = hits[..., 5:8]
    with np.errstate(invalid="ignore", over="ignore"):
        n_sum, a_sum = normal_x[:, 0].copy(), albedo_x[:, 0].copy()
        for s in range(1, spp):
            n_sum = n_sum + normal_x[:, s]
            a_sum = a_sum + albedo_x[:, s]
        if spp > 1:
            inv = np.float32(1) / np.float32(spp)
            n_sum, a_sum = inv * n_sum, inv * a_sum
    return {"id": sphere[:, 0].copy(), "depth": hits[:, 0, 0].copy(), "normal": n_sum.astype(np.float32),
            "albedo": a_sum.astype(np.float32), "coverage": hit.sum(1).astype(np.int32)}


def oracle_gbuffer(oracle, colours, h, w, spp):
    """The rule over the CPU oracle's trace_hits / trace_paths of the frame's camera rays, shaped [h, w, ...]."""
    import raytracers_b200 as R
    rays = R.camera_rays(oracle.camera(), h, w, spp).reshape(-1, 6)
    g = gbuffer_rule(oracle.trace_hits(rays), oracle.trace_paths(rays, max_depth=1)[0], colours, spp)
    return {k: v.reshape((h, w) + v.shape[1:]) for k, v in g.items()}


def gpu_rule(ctx, pr, rays, colours, spp):
    """The rule over the GPU's own trace_hits / trace_paths of camera rays float32 [n, spp, 6]."""
    d = _dev(np.asarray(rays, np.float32).reshape(-1, 6))
    hits = ctx.trace_hits(pr, d)
    buf = np.concatenate([_np(hits["t"])[:, None], _np(hits["sphere"]).view(np.float32)[:, None], _np(hits["p"]),
                          _np(hits["normal"])], 1)
    sky = _np(ctx.trace_paths(pr, d, max_depth=1)[0])
    return gbuffer_rule(buf, sky, colours, spp)


def differ(got, want, what):
    """Asserts that every buffer of `want` is in `got`, equal bit for bit (NaN-aware for the floats)."""
    for k, v in want.items():
        g = np.asarray(got[k])
        if k in ("id", "coverage"):
            bad = int((g.astype(np.int32) != v).sum())
        else:
            bad = bits_differ(g, v)
        assert bad == 0, f"{what}: {k} differs in {bad} values"


def oracle_identities(spheres, cam, h, w, spp, what):
    """The rule on the oracle, checked against the oracle's frame: albedo where coverage == 0, and coverage at spp 1."""
    g = oracle_gbuffer(Q.prepare_custom(spheres, cam, h, w), spheres[:, 3:6], h, w, spp)
    _, rgb, _ = O.Scene.custom(spheres, cam).prepare(h, w).render(h, w, spp, want_rgb=True)
    sky = g["coverage"] == 0
    assert bits_differ(g["albedo"][sky], rgb[sky]) == 0, f"{what}: albedo of uncovered pixels is not the frame"
    if spp == 1:
        assert ((g["coverage"] == 1) == (g["id"] >= 0)).all(), f"{what}: coverage at spp 1"
    assert ((g["id"] >= 0) == (g["depth"] >= 0)).all() and (g["depth"][g["id"] < 0] == -1).all(), what
    assert ((g["coverage"] >= 0) & (g["coverage"] <= spp)).all(), what
    return g


# ------------------------------------------------------------------------------------------ CPU


def _cpu_scene(name):
    if name == "dense":
        return dense_scene(3000)
    return SCENES[name]()


@pytest.mark.parametrize("spp", [1, 3, 8])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "dense"])
def test_rule_on_the_oracle(scene, spp):
    s, c = _cpu_scene(scene)
    h, w = 37, 53
    g = oracle_identities(s, c, h, w, spp, f"{scene} spp {spp}")
    assert (g["coverage"] > 0).any(), "the frame has hits"
    assert scene == "rgbbox" or (g["coverage"] == 0).any(), "the frame has pixels whose samples all leave for the sky"


def test_camera_inside_a_sphere():
    """Every camera ray starts inside sphere 0: its first hit is the far side (t > 0.1), outward normal, full coverage."""
    s = np.float32([[0, 0, 0, 0.3, 0.6, 0.9, 50], [0, 0, -20, 0.9, 0.1, 0.1, 2]])
    c = np.float32([0, 0, 0, 0, 0, -1, 60])
    g = oracle_identities(s, c, 24, 32, 3, "camera inside")
    assert (g["coverage"] == 3).all() and (g["depth"] > 0.1).all()
    assert (g["id"] == 0).sum() > 0 and ((g["id"] == 0) | (g["id"] == 1)).all()


def test_sphere_beyond_2_pow_24():
    """A sphere whose hits lie beyond t = 2^25: t_best + 1 rounds to t_best, so objs_hit's re-intersection in (0, t_best + 1)
    fails and there is no hit: id -1, albedo the sky colour.  A near sphere in the same frame is hit normally."""
    s = np.float32([[0, 0, -1.6e8, 0.2, 0.8, 0.2, 8e7], [1.2, 0, -5, 0.9, 0.5, 0.1, 0.6]])
    c = np.float32([0, 0, 0, 0, 0, -1, 60])
    h, w = 24, 32
    o = Q.prepare_custom(s, c, h, w)
    import raytracers_b200 as R
    rays = R.camera_rays(o.camera(), h, w, 1).reshape(-1, 6)
    # premise: the search finds the far sphere (the occlusion walk accepts it in (0, 1e9)) where the hit query reports none
    occluded = o.trace_occluded(rays, 0.0, 1e9).reshape(h, w)
    g = oracle_identities(s, c, h, w, 1, "far sphere")
    far = occluded & (g["id"] < 0)
    assert far.sum() > h * w // 4, "most of the frame sees the far sphere's failed re-intersection"
    assert (g["coverage"][far] == 0).all() and (g["depth"][far] == -1).all()
    assert (g["id"] == 1).any(), "the near sphere is hit"


def test_nan_camera():
    s, c = SCENES["rgbbox_top_down"]()
    assert np.isnan(Q.prepare_custom(s, c, 24, 32).camera()).any(), "premise: the camera is NaN"
    for spp in (1, 2):
        oracle_identities(s, c, 24, 32, spp, f"NaN camera, spp {spp}")


def test_python_rejects_unknown_outputs(R):
    ctx = object.__new__(R.Context)
    with pytest.raises(ValueError, match="unknown output"):
        R.Context.render_gbuffer(ctx, None, 8, 8, 1, outputs=("id", "position"))
    assert R.QUERIES[8] == "gbuffer"


# ------------------------------------------------------------------------------------------ GPU


def _ctx_scene(R, scene, h, w, **kw):
    ctx = R.Context(device=0, **kw)
    if scene in ("rgbbox", "irreg"):
        sc = ctx.scene(scene)
    elif scene == "dense":
        sc = ctx.scene_from_arrays(*dense_scene(3000))
    else:
        sc = ctx.scene_from_arrays(*ALL_SCENES[scene]())
    return ctx, sc, ctx.prepare_scene(h, w, sc)


def _gb_into(ctx, pr, h, w, spp, names=OUTPUTS):
    """render_gbuffer_into on sentinel-filled buffers of the outputs in `names`: numpy dict"""
    torch = _torch()
    shapes = {"id": (h, w), "depth": (h, w), "normal": (h, w, 3), "albedo": (h, w, 3), "coverage": (h, w)}
    bufs = {k: torch.full(shapes[k], SENTINEL, dtype=torch.int32, device="cuda") for k in names}
    torch.cuda.synchronize()
    ptr = lambda k: bufs[k].data_ptr() if k in bufs else 0
    ctx.render_gbuffer_into(pr, h, w, spp, ptr("id"), ptr("depth"), ptr("normal"), ptr("albedo"), ptr("coverage"))
    ctx.sync()
    return {k: _np(v) if k in ("id", "coverage") else _np(v).view(np.float32) for k, v in bufs.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 3])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "dense"])
def test_small_frames_equal_the_oracle_rule_on_every_subset(R, scene, spp):
    h, w = 37, 53
    s, c = _cpu_scene(scene)
    want = oracle_gbuffer(Q.prepare_custom(s, c, h, w), s[:, 3:6], h, w, spp)
    ctx, sc, pr = _ctx_scene(R, scene, h, w)
    got = ctx.render_gbuffer(pr, h, w, spp)
    assert set(got) == set(OUTPUTS)
    assert got["id"].dtype == _torch().int32 and tuple(got["normal"].shape) == (h, w, 3)
    differ({k: _np(v) for k, v in got.items()}, want, f"{scene} spp {spp}")
    p = ctx.last_plan()
    assert p["query"] == "gbuffer" and p["spread"] == 0 and p["kernel"] == R.KERNELS["warpqueue"]
    for r in range(1, len(OUTPUTS) + 1):
        for names in itertools.combinations(OUTPUTS, r):
            got = _gb_into(ctx, pr, h, w, spp, names)
            differ(got, {k: want[k] for k in names}, f"{scene} spp {spp}, outputs {names}")
    ctx.close()


LARGE = [("rgbbox", 1000, 1000, 1), ("rgbbox", 1000, 1000, 16), ("rgbbox", 1000, 1000, 64), ("irreg", 1000, 1000, 1),
         ("irreg", 1000, 1000, 16), ("irreg", 1000, 1000, 64), ("million", 512, 512, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("scene,h,w,spp", LARGE)
def test_large_frames_equal_the_rule_on_gpu_queries(R, scene, h, w, spp):
    """Sampled rows (every row at one sample) against the rule on the GPU's own trace_hits / trace_paths; where nothing
    is hit, albedo against render_into's float framebuffer."""
    torch = _torch()
    with R.Context(device=0) as ctx:
        sc = ctx.scene_random(1 << 20, 1) if scene == "million" else ctx.scene(scene)
        pr = ctx.prepare_scene(h, w, sc)
        colours = sc.arrays()[0][:, 3:6]
        got = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
        rng = np.random.default_rng(spp)
        rows = np.arange(h) if spp == 1 else np.unique(np.concatenate([[0, 1, h // 2, h - 1], rng.integers(0, h, 40)]))
        js, iss = np.repeat(rows, w), np.tile(np.arange(w), len(rows))
        want = gpu_rule(ctx, pr, _pixel_rays(R, pr.info()["camera"], h, w, js, iss, spp), colours, spp)
        differ({k: v[rows].reshape((-1,) + v.shape[2:]) for k, v in got.items()}, want, f"{scene} {h}x{w} spp {spp}")
        pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
        rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
        ctx.sync()
        sky = got["coverage"] == 0
        assert bits_differ(got["albedo"][sky], _np(rgb)[sky]) == 0
        assert (got["coverage"] > 0).any() and sky.any()
        if spp == 1:
            assert ((got["coverage"] == 1) == (got["id"] >= 0)).all()


def _input_range_cases():
    cases = [(name, sp) for name in ALL_SCENES for sp in (1, 3)]
    return cases + [("comb", 1), ("comb", 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("scene,spp", _input_range_cases())
def test_input_ranges_and_limit_scenes(R, scene, spp):
    """Out-of-range colours, NaN cameras, far-out scenes, degenerate radii and the deepest tree, against the rule on the
    CPU oracle and against the oracle's frame where nothing is hit."""
    if scene == "comb":
        s, c = LS.comb_scene(200)[0], LS.COMB_CAM
        h, w = 48, 64
    else:
        s, c = ALL_SCENES[scene]()
        h, w = frame_size(scene)
    want = oracle_identities(s, c, h, w, spp, f"{scene} spp {spp}")
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        got = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
        differ(got, want, f"{scene} spp {spp}")


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS + [{"wq_packet": 24}, {"wq_packet": 0}, {"wq_spread": 0}], ids=str)
def test_every_plan(R, plan):
    h, w, spp = 203, 301, 5
    ctx, sc, pr = _ctx_scene(R, "irreg", h, w, **plan)
    s, c = sc.arrays()
    want = oracle_gbuffer(Q.prepare_custom(s, c, h, w), s[:, 3:6], h, w, spp)
    differ({k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}, want, str(plan))
    assert ctx.last_plan()["spread"] == 0
    ctx.close()


@pytest.mark.gpu
def test_forced_boundaries(R, forced):
    """Every stage_cap point at K = 1 / 2, with and without the packet walk: the staging split of render_into's
    pixel-bound frame, the rule on the oracle, and exactly the 12 reachable kGBuffer instantiations launched."""
    case, launched = forced["case"], set()
    want = {spp: oracle_gbuffer(case.oracle, case.spheres[:, 3:6], H, W, spp) for spp in (1, 3)}
    for cap_name, cap, nodes, spheres in forced["caps"]:
        for plan in FORCED_PLANS:
            for packet in (0, 8):
                what = f"{cap_name} (stage_cap {cap}), {plan}, wq_packet {packet}"
                with R.Context(device=0, stage_cap=cap, wq_packet=packet, **plan) as ctx:
                    pr = case.prepare(ctx)
                    for spp in (1, 3):
                        got = {k: _np(v) for k, v in ctx.render_gbuffer(pr, H, W, spp).items()}
                        p = ctx.last_plan()
                        expect(p, f"{what}, spp {spp}", query="gbuffer", spread=0, k=plan["wq_k"], warps=plan["wq_warps"],
                               packet=packet, smem_nodes=nodes, smem_spheres=spheres)
                        differ(got, want[spp], f"{what}, spp {spp}")
                        launched.add(variant(p))
    reachable = {("gbuffer", False, k, False, pk, st) for k in (1, 2) for pk in (False, True)
                 for st in ("partial", "nodes", "whole")}
    assert launched == reachable and len(reachable) == 12, sorted(reachable ^ launched)


@pytest.mark.gpu
def test_renders_around_gbuffers_plan_and_launch_as_before(R):
    torch = _torch()
    h, w = 250, 250
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")

    def run(with_gbuffer):
        ctx, _, pr = _ctx_scene(R, "irreg", h, w)
        frames, launches, plans = [], [], []
        for spp in (1, 1, 4, 1, 4):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            launches.append(ctx.launch_count() - n0)
            plans.append(ctx.last_plan())
            frames.append(_np(out))
            if with_gbuffer:
                n0 = ctx.launch_count()
                ctx.render_gbuffer(pr, h, w, spp=4)
                assert ctx.launch_count() - n0 == 1, "one launch: no probe, no order sort"
                assert ctx.last_render_ms() > 0
        ctx.close()
        return frames, launches, plans

    plain, around = run(False), run(True)
    assert plain[1] == around[1] and plain[2] == around[2]
    assert plain[1][0] > 1 and plain[1][1] == 1, "the learned order is recorded by the first frame and used by the second"
    for a, b in zip(plain[0], around[0]):
        assert (a == b).all()


@pytest.mark.gpu
def test_torch_stream_and_freeing_the_scene_in_flight(R):
    torch = _torch()
    h, w, spp = 300, 400, 3
    ctx, sc, pr = _ctx_scene(R, "rgbbox", h, w)
    want = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        got = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
    differ(got, want, "torch stream")
    ctx.set_stream(None)
    s, c = SCENES["rgbbox"]()
    outs = [{k: torch.empty_like(_torch().from_numpy(v)).cuda() for k, v in want.items()} for _ in range(3)]
    torch.cuda.synchronize()
    for o in outs:
        pr2 = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        ctx.render_gbuffer_into(pr2, h, w, spp, *(o[k].data_ptr() for k in OUTPUTS))
        pr2.free()          # while the call may still be in flight
    ctx.sync()
    for o in outs:
        differ({k: _np(v) for k, v in o.items()}, want, "scene freed in flight")
    ctx.close()


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w, spp = 37, 53, 3
    ctx, sc, pr = _ctx_scene(R, "rgbbox", h, w)
    want = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
    buf = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")

    class Freed:
        handle = None

    cases = [(dict(spp=0), "spp must be >= 1"), (dict(h=0), "bad image size"), (dict(w=65537), "bad image size"),
             (dict(prepared=Freed()), "invalid prepared scene"), (dict(shard=(1, 2)), "shard set"),
             (dict(ptr=0), "every output is NULL")]
    for change, message in cases:
        a = dict(h=h, w=w, spp=spp, prepared=pr, shard=None, ptr=buf.data_ptr())
        a.update(change)
        if a["shard"]:
            ctx.set_shard(*a["shard"])
        n0 = ctx.launch_count()
        with pytest.raises(R.RayError, match=message):
            ctx.render_gbuffer_into(a["prepared"], a["h"], a["w"], a["spp"], normal_dev=a["ptr"])
        assert ctx.launch_count() == n0
        ctx.set_shard(0, 1)
        differ({k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}, want, message)
    with pytest.raises(ValueError, match="unknown output"):
        ctx.render_gbuffer(pr, h, w, spp, outputs=("albedo", "position"))
    ctx.close()


@pytest.mark.gpu
def test_outputs_past_4_gib(R):
    """19200 x 19200 pixels: the normal and albedo buffers pass 2^32 bytes.  A single small sphere in view; sampled rows
    against the rule on the GPU's own queries."""
    torch = _torch()
    h = w = 19200
    assert 12 * h * w > 1 << 32
    s = np.float32([[0, 0, 0, 0.9, 0.4, 0.2, 0.6], [0, -2.2, 0, 0.2, 0.4, 0.9, 1.2]])   # the second at the bottom edge
    c = np.float32([0, 0, 3, 0, 0, 0, 40])
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        got = ctx.render_gbuffer(pr, h, w, 1)
        rows = np.array([0, 1, h // 2 - 1, h // 2, h - 2, h - 1])
        sampled = {k: _np(v[torch.from_numpy(rows).cuda()]).reshape((len(rows) * w,) + tuple(v.shape[2:]))
                   for k, v in got.items()}
        del got
        torch.cuda.empty_cache()
        js, iss = np.repeat(rows, w), np.tile(np.arange(w), len(rows))
        want = gpu_rule(ctx, pr, _pixel_rays(R, pr.info()["camera"], h, w, js, iss, 1), s[:, 3:6], 1)
        differ(sampled, want, "19200 x 19200")
        assert (sampled["id"][-w:] >= 0).any(), "the last row, past 4 GiB of normals, sees a sphere"
