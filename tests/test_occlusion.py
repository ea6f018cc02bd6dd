"""Occlusion queries (include/ray_b200.h ray_b200_trace_occluded): is any sphere the BVH walk reaches hit in
(t_min, t_max)?  The answer is an OR over the reached leaves, so the GPU's early-exit traversal must equal the CPU
oracle's full walk bit for bit, whatever its schedule.  The relation with the closest-hit query is checked too: at
t_min = 0.1, occluded equals "trace_hits reports a hit" for every ray whose closest hit has t < 2^24."""
import numpy as np
import pytest

import limit_scenes as LS
import occlusion_oracle as Q   # tests/occlusion_oracle.py: the CPU oracle of the occlusion query
from test_ray_queries import ALONG_Z, TWO_CAM, TWO_SPHERES, random_rays

GiB = 1 << 30
T24 = np.float32(1 << 24)

# ------------------------------------------------------------------------------------------ helpers


def max_hit_t(spheres, rays):
    """An upper bound of every t at which a ray can meet a sphere: a hit point lies on some sphere, so
    t * |d| <= |o - c| + r for that sphere.  Rays with d = 0 never hit (their discriminant is 0)."""
    s = np.asarray(spheres, np.float64)
    r = np.asarray(rays, np.float64)
    dist = np.linalg.norm(r[:, None, :3] - s[None, :, :3], axis=2).max(1) + s[:, 6].max()
    dn = np.linalg.norm(r[:, 3:6], axis=1)
    ok = dn > 0
    return float((dist[ok] / dn[ok]).max()) if ok.any() else 0.0


def light_above(spheres):
    """A point light above the middle of the scene's bounding box, one box height above its top."""
    s = np.asarray(spheres, np.float32)
    lo = (s[:, :3] - s[:, 6:7]).min(0)
    hi = (s[:, :3] + s[:, 6:7]).max(0)
    return np.float32([(lo[0] + hi[0]) / 2, hi[1] + (hi[1] - lo[1]), (lo[2] + hi[2]) / 2])


def segment_rays(points, target):
    """Point-to-point visibility rays: origin = point, direction = target - point (not normalised), so that the
    interval (1e-4, 1 - 1e-4) covers the open segment."""
    p = np.asarray(points, np.float32)
    return np.ascontiguousarray(np.concatenate([p, np.asarray(target, np.float32)[None] - p], 1), np.float32)


SEGMENT = (1e-4, 1 - 1e-4)

# (ray, t_min, t_max, occluded) on the two-sphere scene: A = centre 0, radius 1 (roots 4 and 6 along ALONG_Z),
# B = centre (0, 0, 10), radius 1 (roots 14 and 16)
TWO_SPHERE_CASES = [
    (ALONG_Z, 0.0, 1e9, True),                 # blocked
    (ALONG_Z, 0.0, 3.0, False),                # the segment stops short of A
    (ALONG_Z, 0.0, 4.0, False),                # t_max exactly at root1: strict <, not occluded
    (ALONG_Z, 0.0, 4.0001, True),
    (ALONG_Z, 4.0, 5.0, False),                # t_min exactly at root1: root1 rejected, root2 = 6 outside
    (ALONG_Z, 4.0, 6.5, True),                 # t_min exactly at root1: root2 accepted
    (ALONG_Z, 5.0, 1e9, True),                 # no epsilon: A's root2 at 6 counts, and B behind it
    (ALONG_Z, 6.0, 14.0, False),               # between the spheres, both bounds exactly at roots
    ([0, 0, 0, 1, 0, 0], 0.0, 1e9, True),      # origin inside A: root2 = 1
    ([0, 0, 0, 1, 0, 0], 0.0, 1.0, False),     # ... which is the interval's end
    ([0, 0, -0.5, 0, 0, 1], 0.0, 1.0, False),  # inside A, the exit at 1.5 is beyond the interval
    ([0, 5, 0, 0, 1, 0], 0.0, 1e9, False),     # away from everything
    (ALONG_Z, 3.0, 3.0, False),                # t_max <= t_min
    (ALONG_Z, 50.0, 10.0, False),
]


def two_sphere_results(trace):
    return [bool(trace(np.array([c[0]], np.float32), c[1], c[2])[0]) for c in TWO_SPHERE_CASES]


# ------------------------------------------------------------------------------------------ CPU


def test_occluded_is_bound(R):
    assert "ray_b200_trace_occluded" in set(R.declared_symbols())
    assert hasattr(R.Context, "trace_occluded") and hasattr(R.Context, "trace_occluded_into")


def test_oracle_two_sphere_known_answers():
    pr = Q.prepare_custom(TWO_SPHERES, TWO_CAM, 64, 64)
    got = two_sphere_results(pr.trace_occluded)
    assert got == [c[3] for c in TWO_SPHERE_CASES]


@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_oracle_occlusion_equals_hits_at_epsilon(R, name):
    """occluded(r, 0.1, T) == (trace_hits(r, 0.1, T).t >= 0) while closest hits stay below 2^24."""
    pr = Q.prepare(name, 64, 64)
    spheres, _ = R.host_scene(name)
    rays = random_rays(spheres, 20000, seed=17)
    assert max_hit_t(spheres, rays) < T24     # premise: the re-intersection of trace_hits cannot fail
    for t_max in (1e9, 100.0, 5.0):
        occ = pr.trace_occluded(rays, 0.1, t_max)
        hit = pr.trace_hits(rays, 0.1, t_max)[:, 0] >= 0
        assert int((occ != hit).sum()) == 0, t_max
        assert 0.05 < occ.mean() < 0.95, (t_max, occ.mean())
    # below t_min = 0.1 the two differ by design: occlusion has no epsilon
    occ0 = pr.trace_occluded(rays, 0.0, 1e9)
    assert (occ0 >= pr.trace_occluded(rays, 0.1, 1e9)).all()


def test_segment_rays_of_the_shadow_workload(R):
    """Shadow rays end at the light: every hit point has a segment, and the interval excludes both end points."""
    h, w = 64, 96
    pr = Q.prepare("irreg", h, w)
    spheres, _ = R.host_scene("irreg")
    hits = pr.trace_hits(R.camera_rays(pr.camera(), h, w).reshape(-1, 6))
    p = hits[hits[:, 0] >= 0, 2:5]
    light = light_above(spheres)
    rays = segment_rays(p, light)
    assert rays.shape == (p.shape[0], 6) and p.shape[0] > 100
    np.testing.assert_allclose(rays[:, :3] + rays[:, 3:], np.broadcast_to(light, p.shape), atol=1e-4)  # f32 rounding
    occ = pr.trace_occluded(rays, *SEGMENT)
    assert 0.05 < occ.mean() < 0.95


# ------------------------------------------------------------------------------------------ GPU

def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _gpu_case(R, name, h=500, w=500, n=None, seed=1, **ctx_kw):
    ctx = R.Context(device=0, **ctx_kw)
    sc = ctx.scene(name, n=n, seed=seed)
    return ctx, sc, ctx.prepare_scene(h, w, sc)


def _np(t):
    return t.cpu().numpy()


INTERVALS = [(0.0, 1e9), (0.1, 1e9), (1.0, 100.0), (2.5, 1e9), (40.0, 7.0)]
RANDOM_SCENES = [("rgbbox", None), ("irreg", None), ("random", 30000)]


@pytest.mark.gpu
def test_two_sphere_known_answers_on_gpu(R):
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(64, 64, ctx.scene_from_arrays(TWO_SPHERES, TWO_CAM))
        got = two_sphere_results(lambda r, lo, hi: _np(ctx.trace_occluded(pr, _dev(r), t_min=lo, t_max=hi)))
        assert got == [c[3] for c in TWO_SPHERE_CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_spheres", RANDOM_SCENES)
def test_random_rays_equal_oracle(R, name, n_spheres):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, name, n=n_spheres)
    with ctx:
        rays = random_rays(sc.arrays()[0], 8192, seed=23)
        o = Q.prepare(name, 500, 500, n=n_spheres)
        d = _dev(rays)
        for t_min, t_max in INTERVALS:
            got = ctx.trace_occluded(pr, d, t_min=t_min, t_max=t_max)
            assert got.dtype == torch.bool and got.shape == (rays.shape[0],)
            want = o.trace_occluded(rays, t_min, t_max)
            assert int((_np(got) != want).sum()) == 0, (t_min, t_max)
            if t_max > t_min:
                assert want.any() and not want.all(), (t_min, t_max)   # both answers occur
            else:
                assert not want.any()


@pytest.mark.gpu
def test_random_rays_on_the_million_sphere_scene(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "random", 2000, 2000, n=1000000)
    with ctx:
        assert pr.info()["smem_nodes"] < pr.info()["n_inner"]
        rays = random_rays(sc.arrays()[0], 65536, seed=29)
        d = _dev(rays)
        out = torch.empty((rays.shape[0],), dtype=torch.bool, device="cuda")
        torch.cuda.synchronize()   # the context's own stream is not ordered after torch's
        ctx.trace_occluded_into(d.data_ptr(), rays.shape[0], pr, out.data_ptr(), t_min=0.1)
        ctx.sync()
        sub = slice(0, None, 16)
        o = Q.prepare("random", 2000, 2000, n=1000000)
        want = o.trace_occluded(rays[sub], 0.1, 1e9)
        assert int((_np(out)[sub] != want).sum()) == 0
        assert 0.02 < want.mean() < 0.98


def _shadow_case(R, ctx, sc, pr, h, w):
    """Camera rays through trace_hits, then segments from every hit point to the light."""
    hits = ctx.trace_hits(pr, _dev(R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6)))
    t = _np(hits["t"])
    return segment_rays(_np(hits["p"])[t >= 0], light_above(sc.arrays()[0]))


@pytest.mark.gpu
def test_shadow_rays(R):
    h, w = 500, 500
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        rays = _shadow_case(R, ctx, sc, pr, h, w)
        assert rays.shape[0] > 0.3 * h * w
        d = _dev(rays)
        got = _np(ctx.trace_occluded(pr, d, *SEGMENT))
        want = Q.prepare("irreg", h, w).trace_occluded(rays, *SEGMENT)
        assert int((got != want).sum()) == 0
        assert 0.05 < want.mean() < 0.95
        # the relation with the GPU's own closest-hit query at t_min = 0.1 (every hit t < t_max < 1 < 2^24)
        for t_max in (SEGMENT[1], 1e9):
            if t_max > 1:
                assert max_hit_t(sc.arrays()[0], rays) < T24
            occ = _np(ctx.trace_occluded(pr, d, t_min=0.1, t_max=t_max))
            hit = _np(ctx.trace_hits(pr, d, t_min=0.1, t_max=t_max)["t"]) >= 0
            assert int((occ != hit).sum()) == 0, t_max


PLANS = [{}, {"wq_k": 1}, {"wq_k": 2}, {"wq_warps": 3}, {"wq_warps": 5}, {"stage_cap": 1024}, {"wq_low": -1},
         {"wq_low": 64}, {"wq_ncap": 256}]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_plan_variants_give_identical_results(R, name):
    h, w = 300, 300
    results = []
    for kw in PLANS:
        ctx, sc, pr = _gpu_case(R, name, h, w, **kw)
        with ctx:
            rays = np.concatenate([random_rays(sc.arrays()[0], 3000, seed=31), _shadow_case(R, ctx, sc, pr, h, w)])
            d = _dev(rays)
            results.append([_np(ctx.trace_occluded(pr, d, t_min=lo, t_max=hi)) for lo, hi in ((0.0, 1e9), (1.0, 200.0), SEGMENT)])
    o = Q.prepare(name, h, w)
    want = [o.trace_occluded(rays, lo, hi) for lo, hi in ((0.0, 1e9), (1.0, 200.0), SEGMENT)]
    for kw, got in zip(PLANS, results):
        for k in range(3):
            assert int((got[k] != want[k]).sum()) == 0, (kw, k)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 33, 1 << 22])
def test_batch_sizes(R, n):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        rays = random_rays(sc.arrays()[0], max(n, 1), seed=n + 3)[:n]
        d = _dev(rays) if n else torch.empty((0, 6), dtype=torch.float32, device="cuda")
        before = ctx.launch_count()
        got = ctx.trace_occluded(pr, d, t_min=0.1)
        if n == 0:
            assert ctx.launch_count() == before and got.shape == (0,)
            return
        assert ctx.launch_count() == before + 1
        assert ctx.last_render_ms() > 0
        sub = slice(None) if n < 1000 else slice(0, None, 997)
        want = Q.prepare("irreg", 500, 500).trace_occluded(rays[sub], 0.1, 1e9)
        assert int((_np(got)[sub] != want).sum()) == 0


@pytest.mark.gpu
def test_edge_rays_equal_oracle(R):
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        spheres = sc.arrays()[0]
        o = Q.prepare("rgbbox", 500, 500)
        c, rad = spheres[:, :3], spheres[:, 6:7]
        rays = [[0, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0], [0, 0, 0, 0, -1, 0], [0, 0, 0, 0, 0, 1],   # all-zero, axis-aligned
                [0, 30, 30, 0, -1, -1], [1, 2, 3, -0.0, 0.0, 1], [0, 0, 0, 1, 1, 0], [-30, -30, -30, 1, 1, 1],
                [5, 5, 5, 0, 0, 0], [-40, 0, 0, 1, 0, 0]]
        rays += [[*(c[k] + rad[k] * np.float32([1, 0, 0])), -1, 0.25, 0.5] for k in range(0, 400, 7)]   # on surfaces
        rays += [[*c[k], 0.3, -1, 0.2] for k in range(3, 400, 11)]                                      # inside spheres
        rays += [[*c[k], 0, 0, 0] for k in range(5, 400, 13)]                                           # d = 0 inside
        rays = np.array(rays, np.float32)
        d = _dev(rays)
        for t_min, t_max in ((0.0, 1e9), (0.1, 1e9), (0.0, 0.05), (0.0, 0.5), (1.0, 3.0), *([SEGMENT])):
            got = _np(ctx.trace_occluded(pr, d, t_min=t_min, t_max=t_max))
            assert int((got != o.trace_occluded(rays, t_min, t_max)).sum()) == 0, (t_min, t_max)
        assert not o.trace_occluded(rays[:1])[0]   # the all-zero direction hits nothing


@pytest.mark.gpu
def test_validation_errors_leave_the_context_usable(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 64, seed=3))
        out = torch.empty((64,), dtype=torch.bool, device="cuda")
        rp, op = rays.data_ptr(), out.data_ptr()
        before = ctx.launch_count()
        bad = [lambda: ctx.trace_occluded_into(rp, -1, pr, op),
               lambda: ctx.trace_occluded_into(rp, (1 << 30) + 1, pr, op),
               lambda: ctx.trace_occluded_into(None, 64, pr, op),
               lambda: ctx.trace_occluded_into(rp, 64, pr, None),
               lambda: ctx.trace_occluded_into(rp, 64, pr, op, t_min=-1.0),
               lambda: ctx.trace_occluded_into(rp, 64, pr, op, t_min=float("nan")),
               lambda: ctx.trace_occluded_into(rp, 64, pr, op, t_max=float("nan")),
               lambda: ctx.trace_occluded_into(rp, 64, pr, op, t_max=float("inf")),
               lambda: ctx.trace_occluded_into(rp, 64, pr, op, t_min=float("inf"))]
        for k, call in enumerate(bad):
            with pytest.raises(R.RayError) as e:
                call()
            assert "trace_occluded" in str(e.value), k
        null_scene = type("P", (), {"handle": None})()
        with pytest.raises(R.RayError, match="invalid prepared scene"):
            ctx.trace_occluded_into(rp, 64, null_scene, op)
        with pytest.raises(ValueError):
            ctx.trace_occluded(pr, rays.double())
        with pytest.raises(ValueError):
            ctx.trace_occluded(pr, rays.cpu())
        assert ctx.launch_count() == before
        ctx.trace_occluded_into(rp, 0, pr, None)   # n == 0 does nothing, NULL buffers included
        got = ctx.trace_occluded(pr, rays)
        assert ctx.launch_count() == before + 1
        assert int((_np(got) != Q.prepare("rgbbox", 500, 500).trace_occluded(_np(rays))).sum()) == 0


@pytest.mark.gpu
def test_freed_scene_in_flight_and_frames_unchanged(R, golden):
    torch = _torch()
    pix, _ = golden["rgbbox_500"]
    h, w = pix.shape
    with R.Context(device=0) as ctx:
        ctx.set_stream(torch.cuda.current_stream().cuda_stream)
        ctx.set_pipeline(True)
        sc = ctx.rgbbox()
        frame_scene = ctx.prepare_scene(h, w, sc)
        rays = random_rays(sc.arrays()[0], 20000, seed=5)
        want = Q.prepare("rgbbox", h, w).trace_occluded(rays, 0.1, 50.0)
        frames = [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(4)]
        outs = []
        for k in range(4):
            ctx.render_batch([{"prepared": frame_scene, "h": h, "w": w, "out_dev": frames[k].data_ptr()}])
            q = ctx.prepare_scene(h, w, sc)   # a scene used by one query only, freed while the query is in flight
            d = _dev(rays)
            occ = torch.empty((rays.shape[0],), dtype=torch.bool, device="cuda")
            ctx.trace_occluded_into(d.data_ptr(), rays.shape[0], q, occ.data_ptr(), t_min=0.1, t_max=50.0)
            q.free()
            outs.append((d, occ))
        ctx.sync()
        torch.cuda.synchronize()
        for k in range(4):
            assert int((frames[k].cpu().numpy() != pix).sum()) == 0, k
            assert int((_np(outs[k][1]) != want).sum()) == 0, k
        ctx.set_pipeline(False)
        ctx.set_stream(None)


@pytest.mark.gpu
def test_queries_are_invisible_to_renders(R, golden):
    pix, _ = golden["irreg_500"]
    h, w = pix.shape
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 50000, seed=9))
        for k in range(3):   # frame 0 records the learned claim order; queries sit between every pair of frames
            img = ctx.render(h, w, pr)
            ctx.trace_occluded(pr, rays, t_min=0.5, t_max=100.0)
            ctx.sync()
            assert int((img.values() != pix).sum()) == 0, k


# ------------------------------------------------------------------------------------------ GPU, limits

COMB_M = 1 << 18            # cluster leaves at depth 48 (tests/test_limits.py)
COMB_H, COMB_W = 48, 64


@pytest.mark.gpu
def test_comb_tree_depth_48(R):
    s, first = LS.comb_scene(COMB_M)
    rays = LS.comb_query_rays(122, seed=2)
    o = Q.prepare_custom(s, LS.COMB_CAM, COMB_H, COMB_W)
    # premise: the closest hits are cluster spheres, at the bottom of the depth-48 comb (the host builder's tree equals
    # the oracle's, tests/test_limits.py)
    tree = R.host_lbvh(s)
    _, leaf_depth = LS.leaf_depths(tree)
    assert int(leaf_depth.max()) == 48
    inv = np.empty_like(tree["perm"])
    inv[tree["perm"]] = np.arange(inv.shape[0], dtype=inv.dtype)
    won = o.trace_hits(rays)[:, 1].view(np.int32)
    assert (won >= 0).all() and (leaf_depth[inv[won]] >= 45).all()
    intervals = [(0.0, 1e9), (0.1, 1e9), (1.0, 100.0), (2.5, 1e9), (0.0, 1.5), (4.0, 1e9)]
    want = {iv: o.trace_occluded(rays, *iv) for iv in intervals}
    assert want[(0.0, 1e9)].all() and not want[(0.0, 1.5)].any()
    for kw in (dict(), dict(wq_k=2), dict(wq_ncap=256), dict(stage_cap=1024), dict(wq_low=-1)):
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(COMB_H, COMB_W, ctx.scene_from_arrays(s, LS.COMB_CAM))
            assert pr.info()["max_depth"] == 48
            d = _dev(rays)
            for iv in intervals:
                got = _np(ctx.trace_occluded(pr, d, t_min=iv[0], t_max=iv[1]))
                assert int((got != want[iv]).sum()) == 0, (kw, iv)


N28 = 1 << 28
SENTINEL = 0xA5   # neither 0 nor 1


@pytest.mark.gpu
def test_2pow28_rays(R):
    torch = _torch()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 10 * GiB:
        pytest.skip(f"2^28 occlusion rays need 10 GiB of free device memory; {free / GiB:.1f} GiB are free")
    assert N28 * 24 > 4 * GiB   # premise: byte offsets of the rays pass 4 GiB
    with R.Context() as ctx:
        sc = ctx.irreg()
        pr = ctx.prepare_scene(500, 500, sc)
        spheres = sc.arrays()[0]
        lo = torch.from_numpy((spheres[:, :3] - spheres[:, 6:7]).min(0)).cuda()
        hi = torch.from_numpy((spheres[:, :3] + spheres[:, 6:7]).max(0)).cuda()
        g = torch.Generator(device="cuda").manual_seed(28)
        rays = torch.empty((N28, 6), dtype=torch.float32, device="cuda")
        ext = 0.1 * (hi - lo)
        rays[:, :3] = torch.rand((N28, 3), generator=g, device="cuda") * (hi - lo + 2 * ext) + (lo - ext)
        d = torch.randn((N28, 3), generator=g, device="cuda")
        rays[:, 3:] = d / d.norm(dim=1, keepdim=True)
        del d
        rng = np.random.default_rng(28)
        idx = np.unique(np.concatenate([rng.integers(1 << 27, N28, 6000), np.arange(N28 - 64, N28), rng.integers(0, 1 << 27, 500)]))
        it = torch.from_numpy(idx).cuda()
        sub = rays[it].cpu().numpy()
        out = torch.full((N28,), SENTINEL, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_occluded_into(rays.data_ptr(), N28, pr, out.data_ptr(), t_min=0.1)
        ctx.sync()
        assert bool((out <= 1).all())   # every output written, and each is 0 or 1
        want = Q.prepare("irreg", 500, 500).trace_occluded(sub, 0.1, 1e9)
        assert int((out[it].cpu().numpy().astype(bool) != want).sum()) == 0
        assert 0.02 < want.mean() < 0.98
