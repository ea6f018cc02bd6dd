"""Ray queries whose rays carry their own interval (include/ray_b200.h struct ray_b200_ray, ray_b200_trace_*_ranged):
closest hit, occlusion and multi-hit.  The answer for ray i is exactly what the per-call query returns for that ray alone
with (rays[i].t_min, rays[i].t_max), so every GPU result is compared bit for bit (all 8 words of every record, and the
counts) with the CPU oracle, and with the per-call form where every ray has the same interval.  A ray whose interval the
per-call entry points reject gets the empty answer."""
import ctypes

import numpy as np
import pytest

import ray_query_oracle as Q   # tests/ray_query_oracle.py: the CPU oracle of the per-call and the ranged ray queries
from ray_query_cases import (ALONG_Z, GiB, INTERVALS, PLANS, RANDOM_SCENES, SEGMENT, TWO_CAM, TWO_SPHERES, _dev, _gpu_case,
                             _np, _torch, hits_differ, random_rays)

# ------------------------------------------------------------------------------------------ helpers

KINDS = ("hits", "occluded", "multi")


def oracle(name, h, w, n=None):
    return Q.prepare(name, h, w, n=n)


def oracle_custom(spheres, cam7, h, w):
    return Q.prepare_custom(spheres, cam7, h, w)


def ranged(rays, t_min, t_max):
    """[n, 8] rays (origin, t_min, direction, t_max) from [n, 6] rays and scalar or per-ray bounds."""
    r = np.asarray(rays, np.float32).reshape(-1, 6)
    n = r.shape[0]
    lo = np.broadcast_to(np.asarray(t_min, np.float32), (n,))
    hi = np.broadcast_to(np.asarray(t_max, np.float32), (n,))
    return np.ascontiguousarray(np.concatenate([r[:, :3], lo[:, None], r[:, 3:], hi[:, None]], 1), np.float32)


def records_differ(got, want):
    return hits_differ(np.asarray(got, np.float32).reshape(-1, 8), np.asarray(want, np.float32).reshape(-1, 8))


def assert_same(kind, got, want, what):
    if kind == "hits":
        assert hits_differ(got, want) == 0, what
    elif kind == "occluded":
        assert int((np.asarray(got) != np.asarray(want)).sum()) == 0, what
    else:
        assert records_differ(got[0], want[0]) == 0, what
        assert int((got[1] != want[1]).sum()) == 0, what


def oracle_ranged(o, kind, rays8, k=4):
    if kind == "hits":
        return o.trace_hits_ranged(rays8)
    if kind == "occluded":
        return o.trace_occluded_ranged(rays8)
    return o.trace_multi_hits_ranged(rays8, k)


def oracle_per_call(o, kind, rays6, t_min, t_max, k=4):
    if kind == "hits":
        return o.trace_hits(rays6, t_min, t_max)
    if kind == "occluded":
        return o.trace_occluded(rays6, t_min, t_max)
    return o.trace_multi_hits(rays6, k, t_min, t_max)


def gpu_query(ctx, pr, d, kind, k=4, **interval):
    """A query through the Context's tensor API on [n, 6] (with t_min= / t_max=) or [n, 8] rays, as host arrays: hit
    records [n, 8], occluded [n] bool, or (records [n, k, 8], counts [n])."""
    torch = _torch()
    if kind == "hits":
        out = ctx.trace_hits(pr, d, **interval)
        return _np(torch.cat([out["t"][:, None], out["sphere"].view(torch.float32)[:, None], out["p"], out["normal"]], 1))
    if kind == "occluded":
        return _np(ctx.trace_occluded(pr, d, **interval))
    out = ctx.trace_multi_hits(pr, d, k, **interval)
    buf = torch.cat([out["t"][..., None], out["sphere"].view(torch.float32)[..., None], out["p"], out["normal"]], -1)
    return _np(buf), _np(out["count"])


def random_intervals(spheres, n, seed):
    """Per-ray intervals: half of them rows of INTERVALS, half (t_min, t_min + exponential) on the scale of the scene."""
    s = np.asarray(spheres, np.float32)
    diag = float(np.linalg.norm((s[:, :3] + s[:, 6:7]).max(0) - (s[:, :3] - s[:, 6:7]).min(0)))
    rng = np.random.default_rng(seed)
    rows = np.array(INTERVALS, np.float32)[rng.integers(0, len(INTERVALS), n)]
    lo = np.where(rng.random(n) < 0.2, 0.0, rng.uniform(0.0, 0.5 * diag, n)).astype(np.float32)
    hi = (lo + rng.exponential(0.3 * diag, n)).astype(np.float32)
    pick = rng.random(n) < 0.5
    return np.where(pick, rows[:, 0], lo).astype(np.float32), np.where(pick, rows[:, 1], hi).astype(np.float32)


def four_lights(spheres):
    """Four point lights over the scene: above the middle of each quarter of its bounding box (x, z), a quarter of the
    box's larger horizontal side above its top."""
    s = np.asarray(spheres, np.float32)
    lo, hi = (s[:, :3] - s[:, 6:7]).min(0), (s[:, :3] + s[:, 6:7]).max(0)
    c, ext = (lo + hi) / 2, hi - lo
    y = hi[1] + max(ext[0], ext[2]) / 4
    return np.float32([[c[0] + sx * ext[0] / 4, y, c[2] + sz * ext[2] / 4] for sx in (-1, 1) for sz in (-1, 1)])


LIGHT_T_MIN = 1e-2   # the self-intersection offset of the unit-direction shadow rays, in distance units


def light_rays(points, lights, seed):
    """Shadow rays with unit directions: from every point toward one of the lights, chosen per ray, with the interval
    (LIGHT_T_MIN, distance - 1e-4), all in float32."""
    p = np.asarray(points, np.float32)
    pick = np.random.default_rng(seed).integers(0, len(lights), p.shape[0])
    v = lights[pick] - p
    dist = np.sqrt((v * v).sum(1, dtype=np.float32)).astype(np.float32)
    return ranged(np.concatenate([p, v / dist[:, None]], 1), np.float32(LIGHT_T_MIN), dist - np.float32(1e-4))


INVALID_T_MIN = [-1.0, -np.inf, np.inf, np.nan]
INVALID_T_MAX = [np.nan, np.inf, -np.inf]


def with_invalid(rays6, t_min, t_max):
    """The rays with their intervals, and after each of them a copy with one invalid bound (cycling through
    INVALID_T_MIN with t_max kept, then INVALID_T_MAX with t_min kept).  Returns ([2n, 8] rays, [2n] bool valid)."""
    good = ranged(rays6, t_min, t_max)
    bad = good.copy()
    cases = [(3, v) for v in INVALID_T_MIN] + [(7, v) for v in INVALID_T_MAX]
    for i in range(bad.shape[0]):
        col, v = cases[i % len(cases)]
        bad[i, col] = v
    out = np.empty((2 * good.shape[0], 8), np.float32)
    out[0::2], out[1::2] = good, bad
    valid = np.zeros(out.shape[0], bool)
    valid[0::2] = True
    return out, valid


# Known answers on the two-sphere scene: A = caller index 1, centre 0, radius 1 (roots 4 and 6 along ALONG_Z);
# B = caller index 0, centre (0, 0, 10), radius 1 (roots 14 and 16).  The tables of the per-call tests, answered here in
# one batch whose rays each carry their own interval.
# (ray, t_min, t_max, t, sphere, p, normal) of the closest-hit query
HIT_CASES = [
    (ALONG_Z, 0.0, 1e9, 4.0, 1, (0, 0, -1), (0, 0, -1)),       # front of A
    (ALONG_Z, 5.0, 1e9, -1.0, -1, None, None),                   # the search (epsilon 0.1) takes A at 4; re-intersected
                                                                 # with (5, 5) it fails
    ([0, 0, -1.0625, 0, 0, 1], 0.0, 1e9, 0.0625, 1, (0, 0, -1), (0, 0, -1)),   # re-intersection with t_min 0
    (ALONG_Z, 3.0, 3.0, -1.0, -1, None, None),                   # t_max <= t_min
    (ALONG_Z, 0.0, 3.0, -1.0, -1, None, None),                   # t_max short of A
    ([0, 0, 12, 0, 0, -1], 0.0, 1e9, 1.0, 0, (0, 0, 11), (0, 0, 1)),   # back of B, from behind
    ([0, 5, 0, 0, 1, 0], 0.0, 1e9, -1.0, -1, None, None),        # away from everything
    ([0, 0, 0, 1, 0, 0], 0.0, 1e9, 1.0, 1, (1, 0, 0), (1, 0, 0)),   # origin inside A
]
# (ray, t_min, t_max, occluded) of the occlusion query
OCC_CASES = [
    (ALONG_Z, 0.0, 1e9, True),
    (ALONG_Z, 0.0, 3.0, False),
    (ALONG_Z, 0.0, 4.0, False),                # t_max exactly at root1: strict <
    (ALONG_Z, 0.0, 4.0001, True),
    (ALONG_Z, 4.0, 5.0, False),                # t_min exactly at root1, root2 = 6 outside
    (ALONG_Z, 4.0, 6.5, True),
    (ALONG_Z, 5.0, 1e9, True),                 # no epsilon: A's exit root counts
    (ALONG_Z, 6.0, 14.0, False),               # both bounds exactly at roots
    ([0, 0, 0, 1, 0, 0], 0.0, 1e9, True),      # origin inside A
    ([0, 0, 0, 1, 0, 0], 0.0, 1.0, False),
    ([0, 0, -0.5, 0, 0, 1], 0.0, 1.0, False),
    ([0, 5, 0, 0, 1, 0], 0.0, 1e9, False),
    (ALONG_Z, 3.0, 3.0, False),
    (ALONG_Z, 50.0, 10.0, False),
]
# (ray, t_min, t_max, count, [(t, sphere, p, normal)]) of the multi-hit query, k = MULTI_K
MULTI_K = 2
MULTI_CASES = [
    (ALONG_Z, 0.0, 1e9, 2, [(4, 1, (0, 0, -1), (0, 0, -1)), (14, 0, (0, 0, 9), (0, 0, -1))]),
    (ALONG_Z, 5.0, 1e9, 2, [(6, 1, (0, 0, 1), (0, 0, 1)), (14, 0, (0, 0, 9), (0, 0, -1))]),   # A's exit: no epsilon
    (ALONG_Z, 0.0, 10.0, 1, [(4, 1, (0, 0, -1), (0, 0, -1))]),
    ([0, 0, 0, 1, 0, 0], 0.0, 1e9, 1, [(1, 1, (1, 0, 0), (1, 0, 0))]),                          # origin inside A
    ([0, 0, -0.5, 0, 0, 1], 0.0, 1e9, 2, [(1.5, 1, (0, 0, 1), (0, 0, 1)), (9.5, 0, (0, 0, 9), (0, 0, -1))]),
    (ALONG_Z, 4.0, 14.0, 1, [(6, 1, (0, 0, 1), (0, 0, 1))]),     # bounds exactly at roots
    (ALONG_Z, 0.0, 4.0, 0, []),
    (ALONG_Z, 6.0, 14.0, 0, []),
    ([0, 5, 0, 0, 1, 0], 0.0, 1e9, 0, []),
    (ALONG_Z, 3.0, 3.0, 0, []),
    (ALONG_Z, 50.0, 10.0, 0, []),
    ([0, 0, -20, 0, 0, 1], 20.0, 40.0, 2, [(21, 1, (0, 0, 1), (0, 0, 1)), (29, 0, (0, 0, 9), (0, 0, -1))]),  # t_min inside A
]
EMPTY = [-1.0, np.int32(-1).view(np.float32), 0, 0, 0, 0, 0, 0]


def mixed_batch(cases):
    """[n, 8] rays of a case table, each with its own interval, followed by ALONG_Z with each invalid bound."""
    good = np.array([[*c[0][:3], c[1], *c[0][3:], c[2]] for c in cases], np.float32)
    bad = [ranged([ALONG_Z], v, 1e9)[0] for v in INVALID_T_MIN] + [ranged([ALONG_Z], 0.0, v)[0] for v in INVALID_T_MAX]
    return np.concatenate([good, np.array(bad, np.float32)]), len(bad)


def check_mixed_batch(trace):
    """trace(kind, rays8, k) -> the answers of a ranged query; checks all three tables and the invalid rays."""
    rays, n_bad = mixed_batch(HIT_CASES)
    got = trace("hits", rays, None)
    for j, (_, _, _, t, sph, p, nrm) in enumerate(HIT_CASES):
        want = EMPTY if t < 0 else [t, np.int32(sph).view(np.float32), *p, *nrm]
        assert hits_differ(got[j:j + 1], np.array([want], np.float32)) == 0, (HIT_CASES[j], got[j])
    assert hits_differ(got[-n_bad:], np.tile(np.array(EMPTY, np.float32), (n_bad, 1))) == 0
    rays, n_bad = mixed_batch(OCC_CASES)
    got = trace("occluded", rays, None)
    assert [bool(v) for v in got] == [c[3] for c in OCC_CASES] + [False] * n_bad
    rays, n_bad = mixed_batch(MULTI_CASES)
    rec, counts = trace("multi", rays, MULTI_K)
    assert rec.shape == (rays.shape[0], MULTI_K, 8)
    want = np.tile(np.array(EMPTY, np.float32), (rays.shape[0], MULTI_K, 1))
    for j, (_, _, _, count, hits) in enumerate(MULTI_CASES):
        for m, (t, s, p, n) in enumerate(hits[:MULTI_K]):
            want[j, m] = [t, np.int32(s).view(np.float32), *p, *n]
    assert list(counts) == [c[3] for c in MULTI_CASES] + [0] * n_bad
    assert records_differ(rec, want) == 0


# ------------------------------------------------------------------------------------------ CPU


def test_ray_struct_layout_and_symbols(R):
    lib = R.load_library()
    assert ctypes.sizeof(R.Ray) == lib.ray_b200_ray_size() == 32
    assert [getattr(R.Ray, f).offset for f in ("o", "t_min", "d", "t_max")] == [0, 12, 16, 28]
    assert {"ray_b200_trace_hits_ranged", "ray_b200_trace_occluded_ranged", "ray_b200_trace_multi_hits_ranged",
            "ray_b200_ray_size"} <= set(R.declared_symbols())
    for kind in ("trace_hits", "trace_occluded", "trace_multi_hits"):
        assert hasattr(R.Context, kind + "_ranged_into")
    assert not hasattr(R.Context, "trace_paths_ranged_into")


def test_python_rejects_mixed_interval_arguments_and_bad_shapes(R):
    torch = pytest.importorskip("torch")
    ctx = R.Context.__new__(R.Context)   # argument checks come before any device or library call
    r8, r7 = torch.zeros((4, 8)), torch.zeros((4, 7))
    for call in (lambda **kw: ctx.trace_hits(None, r8, **kw), lambda **kw: ctx.trace_occluded(None, r8, **kw),
                 lambda **kw: ctx.trace_multi_hits(None, r8, 3, **kw)):
        for kw in ({"t_min": 0.1}, {"t_max": 5.0}, {"t_min": 0.0, "t_max": 1e9}):
            with pytest.raises(ValueError, match="carry their own"):
                call(**kw)
    for call in (lambda r: ctx.trace_hits(None, r), lambda r: ctx.trace_occluded(None, r),
                 lambda r: ctx.trace_multi_hits(None, r, 3)):
        with pytest.raises(ValueError, match=r"shape \[n, 6\] or \[n, 8\]"):
            call(r7)
    with pytest.raises(ValueError, match=r"shape \[n, 6\], got"):
        ctx.trace_paths(None, r8)


def test_oracle_two_sphere_mixed_batch():
    o = oracle_custom(TWO_SPHERES, TWO_CAM, 64, 64)
    check_mixed_batch(lambda kind, rays, k: oracle_ranged(o, kind, rays, k))


@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_oracle_uniform_intervals_equal_the_per_call_form(R, name):
    o = oracle(name, 64, 64)
    rays = random_rays(R.host_scene(name)[0], 8000, seed=81)
    for t_min, t_max in INTERVALS:
        r8 = ranged(rays, t_min, t_max)
        for kind in KINDS:
            assert_same(kind, oracle_ranged(o, kind, r8), oracle_per_call(o, kind, rays, t_min, t_max), (t_min, t_max, kind))
    # -0.0 is a valid t_min
    r8 = ranged(rays, np.float32(-0.0), 1e9)
    assert hits_differ(o.trace_hits_ranged(r8), o.trace_hits(rays, 0.0, 1e9)) == 0


# ------------------------------------------------------------------------------------------ GPU


@pytest.mark.gpu
def test_two_sphere_mixed_batch_on_gpu(R):
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(64, 64, ctx.scene_from_arrays(TWO_SPHERES, TWO_CAM))
        check_mixed_batch(lambda kind, rays, k: gpu_query(ctx, pr, _dev(rays), kind, k))


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_spheres", RANDOM_SCENES)
def test_random_per_ray_intervals_equal_oracle(R, name, n_spheres):
    ctx, sc, pr = _gpu_case(R, name, n=n_spheres)
    with ctx:
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, 8192, seed=83)
        r8 = ranged(rays, *random_intervals(spheres, rays.shape[0], seed=83))
        o = oracle(name, 500, 500, n=n_spheres)
        d = _dev(r8)
        hits = gpu_query(ctx, pr, d, "hits")
        assert_same("hits", hits, o.trace_hits_ranged(r8), name)
        occ = gpu_query(ctx, pr, d, "occluded")
        assert_same("occluded", occ, o.trace_occluded_ranged(r8), name)
        assert occ.any() and not occ.all() and (hits[:, 0] >= 0).any()   # (the random scene is sparse: a few % occluded)
        for k in (1, 4, 16):
            want = o.trace_multi_hits_ranged(r8, k)
            assert_same("multi", gpu_query(ctx, pr, d, "multi", k), want, (name, k))
        assert (want[1] > 1).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_uniform_intervals_equal_the_per_call_form(R, name):
    ctx, sc, pr = _gpu_case(R, name)
    with ctx:
        rays = random_rays(sc.arrays()[0], 20000, seed=85)
        d6 = _dev(rays)
        for t_min, t_max in INTERVALS:
            d8 = _dev(ranged(rays, t_min, t_max))
            for kind in KINDS:
                assert_same(kind, gpu_query(ctx, pr, d8, kind), gpu_query(ctx, pr, d6, kind, t_min=t_min, t_max=t_max),
                            (t_min, t_max, kind))


@pytest.mark.gpu
def test_invalid_intervals_give_empty_answers(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, 3000, seed=87)
        r8, valid = with_invalid(rays, *random_intervals(spheres, rays.shape[0], seed=87))
        o = oracle("rgbbox", 500, 500)
        d = _dev(r8)
        before = ctx.launch_count()
        hits = gpu_query(ctx, pr, d, "hits")
        occ = gpu_query(ctx, pr, d, "occluded")
        rec, counts = gpu_query(ctx, pr, d, "multi", 5)
        assert ctx.launch_count() == before + 3   # every call returned 0 and launched
        assert_same("hits", hits, o.trace_hits_ranged(r8), "hits")
        assert_same("occluded", occ, o.trace_occluded_ranged(r8), "occluded")
        assert_same("multi", (rec, counts), o.trace_multi_hits_ranged(r8, 5), "multi")
        bad = ~valid
        assert hits_differ(hits[bad], np.tile(np.array(EMPTY, np.float32), (int(bad.sum()), 1))) == 0
        assert not occ[bad].any() and not counts[bad].any() and (rec[bad][..., 0] == -1).all()
        # the valid rays are unaffected by their invalid neighbours
        good = _dev(r8[valid])
        assert_same("hits", hits[valid], gpu_query(ctx, pr, good, "hits"), "valid rays alone")
        assert (hits[valid][:, 0] >= 0).any() and occ[valid].any()
        # the per-call entry points still reject these values
        buf = torch.empty((rays.shape[0], 8), dtype=torch.float32, device="cuda")
        d6 = _dev(rays)
        for lo, hi in [(v, 1e9) for v in INVALID_T_MIN] + [(0.0, v) for v in INVALID_T_MAX]:
            with pytest.raises(R.RayError, match="interval"):
                ctx.trace_hits_into(d6.data_ptr(), rays.shape[0], pr, buf.data_ptr(), t_min=lo, t_max=hi)
            with pytest.raises(R.RayError, match="interval"):
                ctx.trace_occluded_into(d6.data_ptr(), rays.shape[0], pr, buf.data_ptr(), t_min=lo, t_max=hi)
            with pytest.raises(R.RayError, match="interval"):
                ctx.trace_multi_hits_into(d6.data_ptr(), 1, pr, 1, buf.data_ptr(), None, t_min=lo, t_max=hi)
        # call-level errors stay errors
        with pytest.raises(R.RayError, match=r"k = 65 is outside \[1, 64\]"):
            ctx.trace_multi_hits_ranged_into(d.data_ptr(), 4, pr, 65, buf.data_ptr())
        with pytest.raises(R.RayError, match="NULL device buffer"):
            ctx.trace_hits_ranged_into(None, 4, pr, buf.data_ptr())
        with pytest.raises(R.RayError, match="outside"):
            ctx.trace_occluded_ranged_into(d.data_ptr(), -1, pr, buf.data_ptr())
        with pytest.raises(R.RayError, match="invalid prepared scene"):
            ctx.trace_hits_ranged_into(d.data_ptr(), 4, type("P", (), {"handle": None})(), buf.data_ptr())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_plans_give_identical_results(R, name):
    h, w = 300, 300
    results = []
    for kw in PLANS:
        ctx, sc, pr = _gpu_case(R, name, h, w, **kw)
        with ctx:
            spheres = sc.arrays()[0]
            rays = random_rays(spheres, 4000, seed=89)
            r8 = ranged(rays, *random_intervals(spheres, rays.shape[0], seed=89))
            d = _dev(r8)
            results.append([gpu_query(ctx, pr, d, kind, 8) for kind in KINDS])
    o = oracle(name, h, w)
    want = [oracle_ranged(o, kind, r8, 8) for kind in KINDS]
    for kw, got in zip(PLANS, results):
        for kind, g, wnt in zip(KINDS, got, want):
            assert_same(kind, g, wnt, (kw, kind))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 33, 1 << 22])
def test_batch_sizes(R, n):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, max(n, 1), seed=n + 91)[:n]
        r8 = ranged(rays, *random_intervals(spheres, n, seed=n + 91))
        d = _dev(r8) if n else torch.empty((0, 8), dtype=torch.float32, device="cuda")
        before = ctx.launch_count()
        got = [gpu_query(ctx, pr, d, kind, 4) for kind in KINDS]
        if n == 0:
            assert ctx.launch_count() == before
            assert got[0].shape == (0, 8) and got[1].shape == (0,) and got[2][0].shape == (0, 4, 8)
            for call in (lambda: ctx.trace_hits_ranged_into(None, 0, pr, None), lambda: ctx.trace_occluded_ranged_into(None, 0, pr, None),
                         lambda: ctx.trace_multi_hits_ranged_into(None, 0, pr, 4, None)):
                call()   # n == 0 does nothing, NULL buffers included
            assert ctx.launch_count() == before
            return
        assert ctx.launch_count() == before + 3
        sub = slice(None) if n < 1000 else slice(0, None, 997)
        o = oracle("irreg", 500, 500)
        for kind, g in zip(KINDS, got):
            g = g[sub] if kind != "multi" else (g[0][sub], g[1][sub])
            assert_same(kind, g, oracle_ranged(o, kind, r8[sub], 4), (n, kind))


@pytest.mark.gpu
def test_rays_buffer_alignment(R):
    """struct ray_b200_ray needs 4-byte alignment: a buffer that is not 16-byte aligned is read with 4-byte loads."""
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, 5000, seed=93)
        r8 = ranged(rays, *random_intervals(spheres, rays.shape[0], seed=93))
        n, k = r8.shape[0], 3
        o = oracle("irreg", 500, 500)
        want = [oracle_ranged(o, kind, r8, k) for kind in KINDS]
        for offset in (0, 1, 2, 3):   # floats; 0 = 16-byte aligned
            raw = torch.zeros((n * 8 + 4,), dtype=torch.float32, device="cuda")
            raw[offset:offset + n * 8] = torch.from_numpy(r8.ravel()).cuda()
            ptr = raw.data_ptr() + 4 * offset
            assert (ptr % 16 == 0) == (offset == 0)
            hits = torch.empty((n, 8), dtype=torch.float32, device="cuda")
            occ = torch.empty((n,), dtype=torch.bool, device="cuda")
            rec = torch.empty((n, k, 8), dtype=torch.float32, device="cuda")
            counts = torch.empty((n,), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.trace_hits_ranged_into(ptr, n, pr, hits.data_ptr())
            ctx.trace_occluded_ranged_into(ptr, n, pr, occ.data_ptr())
            ctx.trace_multi_hits_ranged_into(ptr, n, pr, k, rec.data_ptr(), counts.data_ptr())
            ctx.sync()
            for kind, g, wnt in zip(KINDS, (_np(hits), _np(occ), (_np(rec), _np(counts))), want):
                assert_same(kind, g, wnt, (offset, kind))


@pytest.mark.gpu
def test_million_sphere_scene(R):
    ctx, sc, pr = _gpu_case(R, "random", 2000, 2000, n=1000000)
    with ctx:
        assert pr.info()["smem_nodes"] < pr.info()["n_inner"]
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, 65536, seed=95)
        r8 = ranged(rays, *random_intervals(spheres, rays.shape[0], seed=95))
        d = _dev(r8)
        sub = slice(0, None, 16)
        o = oracle("random", 2000, 2000, n=1000000)
        for kind in KINDS:
            g = gpu_query(ctx, pr, d, kind, 4)
            g = g[sub] if kind != "multi" else (g[0][sub], g[1][sub])
            assert_same(kind, g, oracle_ranged(o, kind, r8[sub], 4), kind)


@pytest.mark.gpu
def test_multi_light_shadows_and_two_scene_composition(R):
    h, w = 300, 300
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        spheres = sc.arrays()[0]
        o = oracle("irreg", h, w)
        # shadow rays from the camera rays' hit points, each to one of four lights, unit directions, t_max = distance
        cam = _dev(R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6))
        hit = gpu_query(ctx, pr, cam, "hits")
        assert hits_differ(hit, o.trace_hits(_np(cam))) == 0
        r8 = light_rays(hit[hit[:, 0] >= 0, 2:5], four_lights(spheres), seed=97)
        assert r8.shape[0] > 1000
        occ = gpu_query(ctx, pr, _dev(r8), "occluded")
        assert_same("occluded", occ, o.trace_occluded_ranged(r8), "shadows")
        assert 0.05 < occ.mean() < 0.95
        rec = gpu_query(ctx, pr, _dev(r8), "multi", 4)
        assert_same("multi", rec, o.trace_multi_hits_ranged(r8, 4), "shadow lists")
        # two prepared scenes: irreg (A) and random spheres in irreg's box (B); the closest hit over both traces B only in
        # front of A's hit
        lo, hi = (spheres[:, :3] - spheres[:, 6:7]).min(0), (spheres[:, :3] + spheres[:, 6:7]).max(0)
        rng = np.random.default_rng(97)
        b = np.concatenate([rng.uniform(lo, hi, (3000, 3)), rng.uniform(0, 1, (3000, 3)), rng.uniform(0.05, 0.4, (3000, 1))], 1)
        b = b.astype(np.float32)
        cam7 = np.float32([0, 10, -30, 0, 0, 0, 60])
        pb = ctx.prepare_scene(h, w, ctx.scene_from_arrays(b, cam7))
        ob = oracle_custom(b, cam7, h, w)
        rays = random_rays(spheres, 20000, seed=98)
        ha = gpu_query(ctx, pr, _dev(rays), "hits")
        wa = o.trace_hits(rays)
        assert hits_differ(ha, wa) == 0
        r8 = ranged(rays, 0.0, np.where(wa[:, 0] >= 0, wa[:, 0], np.float32(1e9)))
        hb = gpu_query(ctx, pb, _dev(r8), "hits")
        wb = ob.trace_hits_ranged(r8)
        assert hits_differ(hb, wb) == 0
        in_front = (wb[:, 0] >= 0) & (wa[:, 0] >= 0)
        assert in_front.any() and ((wa[:, 0] >= 0) & (wb[:, 0] < 0)).any() and ((wa[:, 0] < 0) & (wb[:, 0] >= 0)).any()
        assert (wb[in_front, 0] < wa[in_front, 0]).all()


N28 = 1 << 28
SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes


@pytest.mark.gpu
def test_2pow28_ranged_rays(R):
    """2^28 rays of 32 bytes and their 32-byte records: both byte offsets pass 4 GiB."""
    torch = _torch()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * GiB:
        pytest.skip(f"2^28 ranged rays need 24 GiB of free device memory; {free / GiB:.1f} GiB are free")
    assert N28 * 32 > 4 * GiB
    with R.Context() as ctx:
        sc = ctx.irreg()
        pr = ctx.prepare_scene(500, 500, sc)
        spheres = sc.arrays()[0]
        lo = torch.from_numpy((spheres[:, :3] - spheres[:, 6:7]).min(0)).cuda()
        hi = torch.from_numpy((spheres[:, :3] + spheres[:, 6:7]).max(0)).cuda()
        g = torch.Generator(device="cuda").manual_seed(29)
        rays = torch.empty((N28, 8), dtype=torch.float32, device="cuda")
        ext = 0.1 * (hi - lo)
        rays[:, :3] = torch.rand((N28, 3), generator=g, device="cuda") * (hi - lo + 2 * ext) + (lo - ext)
        d = torch.randn((N28, 3), generator=g, device="cuda")
        rays[:, 4:7] = d / d.norm(dim=1, keepdim=True)
        del d
        rays[:, 3] = torch.rand((N28,), generator=g, device="cuda") * 4
        rays[:, 7] = rays[:, 3] + torch.rand((N28,), generator=g, device="cuda") * 40
        rng = np.random.default_rng(29)
        idx = np.unique(np.concatenate([rng.integers(1 << 27, N28, 6000), np.arange(N28 - 64, N28), rng.integers(0, 1 << 27, 500)]))
        it = torch.from_numpy(idx).cuda()
        sub = rays[it].cpu().numpy()
        hits = torch.full((N28, 8), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_hits_ranged_into(rays.data_ptr(), N28, pr, hits.data_ptr())
        ctx.sync()
        assert not bool((hits == SENTINEL).any())
        want = oracle("irreg", 500, 500).trace_hits_ranged(sub)
        assert hits_differ(hits[it].cpu().numpy().view(np.float32), want) == 0
        assert 0.05 < (want[:, 0] > 0).mean() < 0.95


@pytest.mark.gpu
def test_ranged_queries_are_invisible_to_renders(R, golden):
    pix, _ = golden["irreg_500"]
    h, w = pix.shape
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        spheres = sc.arrays()[0]
        rays = random_rays(spheres, 50000, seed=99)
        d = _dev(ranged(rays, *random_intervals(spheres, rays.shape[0], seed=99)))
        for j in range(3):   # frame 0 records the learned claim order; queries sit between every pair of frames
            img = ctx.render(h, w, pr)
            for kind in KINDS:
                gpu_query(ctx, pr, d, kind, 16)
            ctx.sync()
            assert int((img.values() != pix).sum()) == 0, j


def test_segment_form_and_unit_light_rays_agree_on_the_oracle(R):
    """The multi-light workload's rays: unit directions whose t_max is the light's distance reach the light, and the
    segment form of the same rays (direction = light - point, (1e-4, 1 - 1e-4)) is mostly the same answer.  The two
    differ where f32 rounding moves a root across a bound, and their near offsets differ: 1e-4 of the segment's length
    against LIGHT_T_MIN."""
    h, w = 64, 96
    o = oracle("irreg", h, w)
    spheres, _ = R.host_scene("irreg")
    hits = o.trace_hits(R.camera_rays(o.camera(), h, w).reshape(-1, 6))
    p = hits[hits[:, 0] >= 0, 2:5]
    lights = four_lights(spheres)
    r8 = light_rays(p, lights, seed=7)
    np.testing.assert_allclose(np.linalg.norm(r8[:, 4:7], axis=1), 1, atol=1e-6)
    end = r8[:, :3] + (r8[:, 7:8] + np.float32(1e-4)) * r8[:, 4:7]
    pick = np.random.default_rng(7).integers(0, 4, p.shape[0])
    np.testing.assert_allclose(end, lights[pick], atol=1e-3)
    seg = ranged(np.concatenate([p, lights[pick] - p], 1), SEGMENT[0], SEGMENT[1])
    a, b = o.trace_occluded_ranged(r8), o.trace_occluded_ranged(seg)
    assert 0.05 < a.mean() < 0.95 and (a == b).mean() > 0.99
