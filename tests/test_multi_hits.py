"""Multi-hit queries (include/ray_b200.h ray_b200_trace_multi_hits): the k nearest spheres the BVH walk reaches that a
ray hits in (t_min, t_max), in ascending (t, Morton-sorted leaf), and how many there are.  The set of reached leaves does
not depend on the traversal order, so every record (all 8 words) and every count of the GPU must equal the CPU oracle's
full walk bit for bit, whatever the schedule.  Two identities are checked too: count > 0 equals the occlusion query, and
at t_min = 0.1 record 0 equals the closest-hit record for every ray whose closest hit has t < 2^24."""
import numpy as np
import pytest

import limit_scenes as LS
import ray_query_oracle as Q   # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from ray_query_cases import (ALONG_Z, GiB, INTERVALS, PLANS, RANDOM_SCENES, SEGMENT, T24, TWO_CAM, TWO_SPHERES, _dev,
                             _gpu_case, _np, _shadow_case, _torch, hits_differ, max_hit_t, random_rays)

# ------------------------------------------------------------------------------------------ helpers


def records_differ(got, want):
    """[n, k, 8] hit records: the sphere column as int32, the rest by bits."""
    return hits_differ(np.asarray(got, np.float32).reshape(-1, 8), np.asarray(want, np.float32).reshape(-1, 8))


def gpu_records(out):
    """The dict of Context.trace_multi_hits as ([n, k, 8] float32 records, [n] int32 counts) on the host."""
    torch = _torch()
    buf = torch.cat([out["t"][..., None], out["sphere"].view(torch.float32)[..., None], out["p"], out["normal"]], -1)
    return _np(buf), _np(out["count"])


def gpu_multi(ctx, pr, rays_dev, k, t_min=0.0, t_max=1e9):
    return gpu_records(ctx.trace_multi_hits(pr, rays_dev, k, t_min=t_min, t_max=t_max))


def assert_equal(got, want, what):
    assert records_differ(got[0], want[0]) == 0, what
    assert int((got[1] != want[1]).sum()) == 0, what


def max_hit_t_box(spheres, rays):
    """An upper bound of every t at which a ray can meet a sphere, linear in the ray count: a hit point lies in the
    scene's bounding box (radii included), so t * |d| <= the distance from the origin to the box's farthest corner."""
    s = np.asarray(spheres, np.float64)
    r = np.asarray(rays, np.float64)
    lo, hi = (s[:, :3] - s[:, 6:7]).min(0), (s[:, :3] + s[:, 6:7]).max(0)
    far = np.linalg.norm(np.maximum(np.abs(r[:, :3] - lo), np.abs(r[:, :3] - hi)), axis=1)
    dn = np.linalg.norm(r[:, 3:6], axis=1)
    ok = dn > 0
    return float((far[ok] / dn[ok]).max()) if ok.any() else 0.0


def assert_well_formed(rec, counts, leaf_of_sphere):
    """Records strictly increasing in (t, leaf) up to min(count, k), empty records after them."""
    k = rec.shape[1]
    t = rec[..., 0]
    sphere = rec[..., 1].view(np.int32)
    m = np.minimum(counts, k)
    filled = np.arange(k)[None, :] < m[:, None]
    assert (t[filled] >= 0).all() and (sphere[filled] >= 0).all()
    assert (t[~filled] == -1).all() and (sphere[~filled] == -1).all() and (rec[~filled][:, 2:] == 0).all()
    leaf = np.where(filled, leaf_of_sphere[np.where(filled, sphere, 0)], -1).astype(np.int64)
    # (t, leaf) as one 64-bit key: bits(t) << 32 | leaf, t >= 0 so bit order is numeric order
    key = (t.view(np.uint32).astype(np.int64) << 32) | leaf
    both = filled[:, 1:]
    assert (key[:, 1:][both] > key[:, :-1][both]).all()


# (ray, t_min, t_max, k, count, [(t, sphere, p, normal)]) on the two-sphere scene: A = caller index 1, centre 0,
# radius 1 (roots 4 and 6 along ALONG_Z); B = caller index 0, centre (0, 0, 10), radius 1 (roots 14 and 16)
TWO_SPHERE_CASES = [
    (ALONG_Z, 0.0, 1e9, 2, 2, [(4, 1, (0, 0, -1), (0, 0, -1)), (14, 0, (0, 0, 9), (0, 0, -1))]),
    (ALONG_Z, 5.0, 1e9, 2, 2, [(6, 1, (0, 0, 1), (0, 0, 1)), (14, 0, (0, 0, 9), (0, 0, -1))]),   # A's exit: no epsilon
    (ALONG_Z, 0.0, 10.0, 2, 1, [(4, 1, (0, 0, -1), (0, 0, -1))]),
    (ALONG_Z, 0.0, 1e9, 1, 2, [(4, 1, (0, 0, -1), (0, 0, -1))]),                                   # truncated, full count
    (ALONG_Z, 0.0, 1e9, 5, 2, [(4, 1, (0, 0, -1), (0, 0, -1)), (14, 0, (0, 0, 9), (0, 0, -1))]),
    ([0, 0, 0, 1, 0, 0], 0.0, 1e9, 2, 1, [(1, 1, (1, 0, 0), (1, 0, 0))]),                          # origin inside A
    ([0, 0, -0.5, 0, 0, 1], 0.0, 1e9, 3, 2, [(1.5, 1, (0, 0, 1), (0, 0, 1)), (9.5, 0, (0, 0, 9), (0, 0, -1))]),
    (ALONG_Z, 4.0, 14.0, 2, 1, [(6, 1, (0, 0, 1), (0, 0, 1))]),     # bounds exactly at roots: strict <
    (ALONG_Z, 0.0, 4.0, 2, 0, []),
    (ALONG_Z, 6.0, 14.0, 2, 0, []),
    ([0, 5, 0, 0, 1, 0], 0.0, 1e9, 2, 0, []),                        # away from everything
    (ALONG_Z, 3.0, 3.0, 2, 0, []),                                   # t_max <= t_min
    (ALONG_Z, 50.0, 10.0, 4, 0, []),
]


def check_two_sphere(trace):
    """trace(rays [1, 6], k, t_min, t_max) -> (records [1, k, 8], counts [1])"""
    for case in TWO_SPHERE_CASES:
        ray, lo, hi, k, count, hits = case
        rec, counts = trace(np.array([ray], np.float32), k, lo, hi)
        assert rec.shape == (1, k, 8) and counts.shape == (1,), case
        assert int(counts[0]) == count, case
        want = np.zeros((1, k, 8), np.float32)
        want[0, :, 0] = -1
        want[0, :, 1] = np.int32(-1).view(np.float32)
        for j, (t, s, p, n) in enumerate(hits):
            want[0, j] = [t, np.int32(s).view(np.float32), *p, *n]
        assert records_differ(rec, want) == 0, (case, rec)


# ------------------------------------------------------------------------------------------ CPU


def test_multi_hits_is_bound(R):
    assert "ray_b200_trace_multi_hits" in set(R.declared_symbols())
    assert hasattr(R.Context, "trace_multi_hits") and hasattr(R.Context, "trace_multi_hits_into")


def test_oracle_two_sphere_known_answers():
    pr = Q.prepare_custom(TWO_SPHERES, TWO_CAM, 64, 64)
    check_two_sphere(lambda r, k, lo, hi: pr.trace_multi_hits(r, k, lo, hi))


@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_oracle_self_consistency(R, name):
    pr = Q.prepare(name, 64, 64)
    occ = Q.prepare(name, 64, 64)
    spheres, _ = R.host_scene(name)
    perm = pr.perm(spheres.shape[0])
    leaf_of_sphere = np.empty_like(perm)
    leaf_of_sphere[perm] = np.arange(perm.shape[0], dtype=perm.dtype)
    rays = random_rays(spheres, 20000, seed=41)
    assert max_hit_t(spheres, rays) < T24     # premise of identity 2: the re-intersection of trace_hits cannot fail
    checked = 0
    for t_min, t_max in ((0.0, 1e9), (0.1, 1e9), (1.0, 100.0), (0.1, 20.0)):
        r4, c4 = pr.trace_multi_hits(rays, 4, t_min, t_max)
        r16, c16 = pr.trace_multi_hits(rays, 16, t_min, t_max)
        assert (c4 == c16).all()
        assert records_differ(r16[:, :4], r4) == 0, (t_min, t_max)           # k = 4 is the prefix of k = 16
        assert_well_formed(r4, c4, leaf_of_sphere)
        assert_well_formed(r16, c16, leaf_of_sphere)
        assert (c4 > 4).any(), (t_min, t_max)                                  # some lists are truncated
        # identity 1: count > 0 is the occlusion query
        o = occ.trace_occluded(rays, t_min, t_max)
        assert 0.05 < o.mean() < 0.95, (t_min, t_max, o.mean())
        assert int(((c4 > 0) != o).sum()) == 0, (t_min, t_max)
        # identity 2: at t_min = 0.1 record 0 is the closest-hit record
        if t_min == 0.1:
            assert hits_differ(r4[:, 0], pr.trace_hits(rays, t_min, t_max)) == 0, t_max
            checked += 1
    assert checked == 2
    _, c0 = pr.trace_multi_hits(rays, 1, 0.0, 1e9)
    _, c1 = pr.trace_multi_hits(rays, 1, 0.1, 1e9)
    assert (c0 >= c1).all()   # no epsilon: (0, 0.1) can only add leaves


# ------------------------------------------------------------------------------------------ GPU

KS = [1, 3, 8, 64]


@pytest.mark.gpu
def test_two_sphere_known_answers_on_gpu(R):
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(64, 64, ctx.scene_from_arrays(TWO_SPHERES, TWO_CAM))
        check_two_sphere(lambda r, k, lo, hi: gpu_multi(ctx, pr, _dev(r), k, lo, hi))


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_spheres", RANDOM_SCENES)
def test_random_rays_equal_oracle(R, name, n_spheres):
    ctx, sc, pr = _gpu_case(R, name, n=n_spheres)
    with ctx:
        rays = random_rays(sc.arrays()[0], 8192, seed=43)
        o = Q.prepare(name, 500, 500, n=n_spheres)
        d = _dev(rays)
        several = False
        for t_min, t_max in INTERVALS:
            for k in KS:
                got = gpu_multi(ctx, pr, d, k, t_min, t_max)
                assert got[0].shape == (rays.shape[0], k, 8) and got[1].dtype == np.int32
                want = o.trace_multi_hits(rays, k, t_min, t_max)
                assert_equal(got, want, (t_min, t_max, k))
            if t_max > t_min:
                assert (want[1] > 0).any() and (want[1] == 0).any(), (t_min, t_max)
                several |= bool((want[1] > 1).any())
            else:
                assert not want[1].any()
        assert several   # some rays cross more than one sphere


@pytest.mark.gpu
def test_random_rays_on_the_million_sphere_scene(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "random", 2000, 2000, n=1000000)
    with ctx:
        rays = random_rays(sc.arrays()[0], 65536, seed=47)
        d = _dev(rays)
        k = 4
        hits = torch.empty((rays.shape[0], k, 8), dtype=torch.float32, device="cuda")
        counts = torch.empty((rays.shape[0],), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()   # the context's own stream is not ordered after torch's
        ctx.trace_multi_hits_into(d.data_ptr(), rays.shape[0], pr, k, hits.data_ptr(), counts.data_ptr(), t_min=0.1)
        ctx.sync()
        plan = ctx.last_plan()
        assert plan["query"] == "multihit" and plan["smem_nodes"] < plan["n_inner"] and not plan["all_nodes"], plan
        sub = slice(0, None, 16)
        want = Q.prepare("random", 2000, 2000, n=1000000).trace_multi_hits(rays[sub], k, 0.1, 1e9)
        assert_equal((_np(hits)[sub], _np(counts)[sub]), want, "1M")
        assert (want[1] > k).any() and 0.02 < (want[1] > 0).mean() < 0.98


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_plan_variants_give_identical_results(R, name):
    h, w = 300, 300
    intervals = ((0.0, 1e9), (1.0, 200.0), SEGMENT)
    results = []
    for kw in PLANS:
        ctx, sc, pr = _gpu_case(R, name, h, w, **kw)
        with ctx:
            rays = np.concatenate([random_rays(sc.arrays()[0], 3000, seed=53), _shadow_case(R, ctx, sc, pr, h, w)])
            d = _dev(rays)
            results.append([gpu_multi(ctx, pr, d, k, lo, hi) for lo, hi in intervals for k in (1, 8)])
    o = Q.prepare(name, h, w)
    want = [o.trace_multi_hits(rays, k, lo, hi) for lo, hi in intervals for k in (1, 8)]
    for kw, got in zip(PLANS, results):
        for j in range(len(want)):
            assert_equal(got[j], want[j], (kw, j))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 33, 1 << 22])
def test_batch_sizes(R, n):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        rays = random_rays(sc.arrays()[0], max(n, 1), seed=n + 5)[:n]
        d = _dev(rays) if n else torch.empty((0, 6), dtype=torch.float32, device="cuda")
        before = ctx.launch_count()
        got = gpu_multi(ctx, pr, d, 4, t_min=0.1)
        if n == 0:
            assert ctx.launch_count() == before and got[0].shape == (0, 4, 8) and got[1].shape == (0,)
            return
        assert ctx.launch_count() == before + 1
        assert ctx.last_render_ms() > 0
        sub = slice(None) if n < 1000 else slice(0, None, 997)
        want = Q.prepare("irreg", 500, 500).trace_multi_hits(rays[sub], 4, 0.1, 1e9)
        assert_equal((got[0][sub], got[1][sub]), want, n)


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
        for t_min, t_max in ((0.0, 1e9), (0.1, 1e9), (0.0, 0.05), (0.0, 0.5), (1.0, 3.0), SEGMENT):
            for k in (1, 8):
                assert_equal(gpu_multi(ctx, pr, d, k, t_min, t_max), o.trace_multi_hits(rays, k, t_min, t_max), (t_min, t_max, k))
        assert o.trace_multi_hits(rays[:1], 1)[1][0] == 0   # the all-zero direction hits nothing


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_identities_against_the_other_queries(R, name):
    h, w = 500, 500
    ctx, sc, pr = _gpu_case(R, name, h, w)
    with ctx:
        rays = np.concatenate([random_rays(sc.arrays()[0], 20000, seed=59), _shadow_case(R, ctx, sc, pr, h, w)])
        assert max_hit_t_box(sc.arrays()[0], rays) < T24   # premise of identity 2
        d = _dev(rays)
        checked = 0
        for t_min, t_max in ((0.0, 1e9), (0.1, 1e9), (0.1, 30.0), (2.5, 1e9), SEGMENT, (40.0, 7.0)):
            rec, counts = gpu_multi(ctx, pr, d, 3, t_min, t_max)
            occ = _np(ctx.trace_occluded(pr, d, t_min=t_min, t_max=t_max))
            assert int(((counts > 0) != occ).sum()) == 0, (t_min, t_max)   # identity 1
            if t_max > t_min:
                assert 0.01 < occ.mean() < 0.99, (t_min, t_max)   # both answers occur
            if t_min == 0.1:                                                 # identity 2
                checked += 1
                hits = ctx.trace_hits(pr, d, t_min=t_min, t_max=t_max)
                want = np.concatenate([_np(hits["t"])[:, None], _np(hits["sphere"]).view(np.float32)[:, None],
                                       _np(hits["p"]), _np(hits["normal"])], 1)
                assert hits_differ(rec[:, 0], want) == 0, t_max
        assert checked == 2


@pytest.mark.gpu
def test_tie_groups_keep_the_lowest_caller_indices(R):
    """Coincident groups of up to 100 copies with k = 64: the truncated list is the 64 lowest caller indices at equal t,
    and the count is the whole group, on every plan: no schedule may leak into the result."""
    s, groups = LS.tie_groups()
    rays = LS.tie_rays(len(groups))
    o = Q.prepare_custom(s, LS.TIE_CAM, 96, 128)
    k = 64
    want = o.trace_multi_hits(rays, k)
    assert max(len(g) for g in groups) > k   # premise: some list is truncated
    for g, members in enumerate(groups):
        for r in (5 * g, 5 * g + 1, 5 * g + 3):   # +z, -z, -y: only this group lies on the ray
            m = min(k, len(members))
            assert want[1][r] == len(members), (g, r)
            assert (want[0][r, :m, 0] == 4).all() and (want[0][r, :m, 1].view(np.int32) == members[:m]).all(), (g, r)
    for kw in (dict(), dict(wq_k=1), dict(wq_k=2), dict(stage_cap=1024), dict(wq_warps=3)):
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(96, 128, ctx.scene_from_arrays(s, LS.TIE_CAM))
            d = _dev(rays)
            assert_equal(gpu_multi(ctx, pr, d, k), want, kw)
            assert_equal(gpu_multi(ctx, pr, d, 3, 0.0, 30.0), o.trace_multi_hits(rays, 3, 0.0, 30.0), kw)


@pytest.mark.gpu
def test_comb_tree_depth_48(R):
    s, _ = LS.comb_scene(1 << 18)
    rays = LS.comb_query_rays(122, seed=3)
    o = Q.prepare_custom(s, LS.COMB_CAM, 48, 64)
    intervals = [(0.0, 1e9), (0.1, 1e9), (1.0, 100.0), (0.0, 1.5)]
    want = {(iv, k): o.trace_multi_hits(rays, k, *iv) for iv in intervals for k in (1, 8)}
    assert (want[((0.0, 1e9), 8)][1] > 0).all() and not want[((0.0, 1.5), 8)][1].any()
    for kw in (dict(), dict(wq_k=2), dict(wq_ncap=256), dict(stage_cap=1024)):
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(48, 64, ctx.scene_from_arrays(s, LS.COMB_CAM))
            assert pr.info()["max_depth"] == 48
            d = _dev(rays)
            for (iv, k), w in want.items():
                assert_equal(gpu_multi(ctx, pr, d, k, *iv), w, (kw, iv, k))


N22 = 1 << 22
SENTINEL = 0x7FC0DEAD   # a NaN pattern no record word can take


@pytest.mark.gpu
def test_records_past_4GiB(R):
    torch = _torch()
    k = 64
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * GiB:
        pytest.skip(f"2^22 rays x 64 records need 12 GiB of free device memory; {free / GiB:.1f} GiB are free")
    assert N22 * k * 32 > 4 * GiB   # premise: record byte offsets pass 4 GiB
    with R.Context() as ctx:
        sc = ctx.irreg()
        pr = ctx.prepare_scene(500, 500, sc)
        rays = random_rays(sc.arrays()[0], N22, seed=61)
        d = _dev(rays)
        hits = torch.full((N22, k, 8), SENTINEL, dtype=torch.int32, device="cuda")
        counts = torch.full((N22,), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_multi_hits_into(d.data_ptr(), N22, pr, k, hits.data_ptr(), counts.data_ptr())
        ctx.sync()
        assert not bool((counts == SENTINEL).any())
        assert not bool((hits == SENTINEL).any(dim=2).any())
        rng = np.random.default_rng(61)
        idx = np.unique(np.concatenate([rng.integers(0, N22, 3000), np.arange(N22 - 64, N22)]))
        it = torch.from_numpy(idx).cuda()
        got = (hits[it].cpu().numpy().view(np.float32), counts[it].cpu().numpy())
        want = Q.prepare("irreg", 500, 500).trace_multi_hits(rays[idx], k)
        assert_equal(got, want, "past 4 GiB")
        assert (want[1] > 1).any()


@pytest.mark.gpu
def test_validation_errors_leave_the_context_usable(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 64, seed=7))
        hits = torch.empty((64, 64, 8), dtype=torch.float32, device="cuda")
        counts = torch.empty((64,), dtype=torch.int32, device="cuda")
        rp, hp, cp = rays.data_ptr(), hits.data_ptr(), counts.data_ptr()
        before = ctx.launch_count()
        bad = [lambda: ctx.trace_multi_hits_into(rp, 64, pr, 0, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, 65, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, -1, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, 4, None, cp),
               lambda: ctx.trace_multi_hits_into(None, 64, pr, 4, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, -1, pr, 4, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, (1 << 30) + 1, pr, 4, hp, cp),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, 4, hp, cp, t_min=-1.0),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, 4, hp, cp, t_min=float("nan")),
               lambda: ctx.trace_multi_hits_into(rp, 64, pr, 4, hp, cp, t_max=float("inf"))]
        for j, call in enumerate(bad):
            with pytest.raises(R.RayError) as e:
                call()
            assert "trace_multi_hits" in str(e.value), j
        with pytest.raises(R.RayError, match=r"k = 65 is outside \[1, 64\]"):
            ctx.trace_multi_hits_into(rp, 64, pr, 65, hp, cp)
        null_scene = type("P", (), {"handle": None})()
        with pytest.raises(R.RayError, match="invalid prepared scene"):
            ctx.trace_multi_hits_into(rp, 64, null_scene, 4, hp, cp)
        with pytest.raises(ValueError):
            ctx.trace_multi_hits(pr, rays.double(), 4)
        assert ctx.launch_count() == before
        ctx.trace_multi_hits_into(rp, 0, pr, 4, None, None)   # n == 0 does nothing, NULL buffers included
        assert ctx.launch_count() == before
        o = Q.prepare("rgbbox", 500, 500)
        ctx.trace_multi_hits_into(rp, 64, pr, 64, hp, None)   # counts are optional
        ctx.sync()
        assert records_differ(_np(hits), o.trace_multi_hits(_np(rays), 64)[0]) == 0
        got = gpu_multi(ctx, pr, rays, 5, 0.5, 60.0)
        assert ctx.launch_count() == before + 2
        assert_equal(got, o.trace_multi_hits(_np(rays), 5, 0.5, 60.0), "after the errors")


@pytest.mark.gpu
def test_records_at_4_byte_alignment(R):
    """struct ray_b200_hit needs only 4-byte alignment: a buffer that is not 16-byte aligned takes 4-byte stores."""
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        rays = random_rays(sc.arrays()[0], 5000, seed=73)
        d = _dev(rays)
        k = 5
        want = Q.prepare("irreg", 500, 500).trace_multi_hits(rays, k, 0.1, 1e9)
        for offset in (1, 2, 3):   # floats
            raw = torch.empty((rays.shape[0] * k * 8 + 4,), dtype=torch.float32, device="cuda")
            counts = torch.empty((rays.shape[0],), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.trace_multi_hits_into(d.data_ptr(), rays.shape[0], pr, k, raw.data_ptr() + 4 * offset, counts.data_ptr(), t_min=0.1)
            ctx.sync()
            got = _np(raw)[offset:offset + rays.shape[0] * k * 8].reshape(-1, k, 8)
            assert_equal((got, _np(counts)), want, offset)


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
        rays = random_rays(sc.arrays()[0], 20000, seed=67)
        k = 6
        want = Q.prepare("rgbbox", h, w).trace_multi_hits(rays, k, 0.1, 50.0)
        frames = [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(4)]
        outs = []
        for j in range(4):
            ctx.render_batch([{"prepared": frame_scene, "h": h, "w": w, "out_dev": frames[j].data_ptr()}])
            q = ctx.prepare_scene(h, w, sc)   # a scene used by one query only, freed while the query is in flight
            d = _dev(rays)
            hits = torch.empty((rays.shape[0], k, 8), dtype=torch.float32, device="cuda")
            counts = torch.empty((rays.shape[0],), dtype=torch.int32, device="cuda")
            ctx.trace_multi_hits_into(d.data_ptr(), rays.shape[0], q, k, hits.data_ptr(), counts.data_ptr(), t_min=0.1, t_max=50.0)
            q.free()
            outs.append((d, hits, counts))
        ctx.sync()
        torch.cuda.synchronize()
        for j in range(4):
            assert int((frames[j].cpu().numpy() != pix).sum()) == 0, j
            assert_equal((_np(outs[j][1]), _np(outs[j][2])), want, j)
        ctx.set_pipeline(False)
        ctx.set_stream(None)


@pytest.mark.gpu
def test_queries_are_invisible_to_renders(R, golden):
    pix, _ = golden["irreg_500"]
    h, w = pix.shape
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 50000, seed=71))
        for j in range(3):   # frame 0 records the learned claim order; queries sit between every pair of frames
            img = ctx.render(h, w, pr)
            ctx.trace_multi_hits(pr, rays, 16, t_min=0.5, t_max=100.0)
            ctx.sync()
            assert int((img.values() != pix).sum()) == 0, j
