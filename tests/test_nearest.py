"""Nearest-sphere queries (include/ray_b200.h "nearest-sphere queries"): the k nearest spheres to each point, with r an
upper limit on the distance that may be +inf.

The oracle is a brute force over every sphere of a scene in numpy float32, with the header's operation order, as in
test_proximity.py but with r = +inf accepted: numpy's float32 ufuncs round every operation to nearest and np.sqrt on
float32 is correctly rounded, as the kernel's __fsqrt_rn is.  Every GPU output must equal it bit for bit: the bits of d,
sphere indices, and the padding records.

- CPU: the oracle against scipy's float64 k-d tree on equal-radius scenes away from ties, its ordering and padding
  (records at d = +inf included), the Python argument checks, the struct sizes and the declared symbols.
- GPU: built-in, random, limit, input-range and coincident-copy scenes at k = 1, 2, 8, 9 and 64 with unbounded and finite
  balls, inside, on and far outside the scene, and invalid balls; every sphere's own centre at k + 1 (the neighbour
  graph recipe of the header); the identity with query_spheres for finite r; ties at the k-th distance on lattices and
  coincident copies, nested spheres that make d_k negative; scenes far from the origin with tiny radii, huge spheres and
  distances that overflow; stale boxes before and after updates; uniform and ragged batches against their members;
  guarded outputs, errors, stream order and scenes freed or updated with a query in flight.
"""
import ctypes as C

import numpy as np
import pytest

import limit_scenes as LS
import raytracers_b200 as RB
import test_proximity as TP   # the scenes of the proximity tests (input-range, limit and built-in scenes)

KS = (1, 2, 8, 9, 64)
F32 = np.float32
INF = F32(np.inf)

# ------------------------------------------------------------------------------------------ the oracle


def sphere_ok(spheres):
    """Which spheres can be reported: finite centre and radius, radius >= 0 (-0.0 included)"""
    s = np.asarray(spheres, F32)
    with np.errstate(invalid="ignore"):
        return np.isfinite(s[:, :3]).all(1) & np.isfinite(s[:, 6]) & (s[:, 6] >= 0)


def ball_ok(balls):
    """Which balls are valid: finite centre, r >= 0 with r = +inf allowed (NaN and negative r are not)"""
    b = np.asarray(balls, F32)
    with np.errstate(invalid="ignore"):
        return np.isfinite(b[:, :3]).all(1) & (b[:, 3] >= 0)


def distances(spheres, centres):
    """d[q, j] = sqrtf((dx*dx + dy*dy) + dz*dz) - rho in float32, dx = p.x - c.x, for every ball centre and sphere"""
    s = np.asarray(spheres, F32)
    c = np.asarray(centres, F32)
    with np.errstate(all="ignore"):
        dx = s[None, :, 0] - c[:, None, 0]
        dy = s[None, :, 1] - c[:, None, 1]
        dz = s[None, :, 2] - c[:, None, 2]
        return np.sqrt((dx * dx + dy * dy) + dz * dz) - s[None, :, 6]


def brute(spheres, balls, k=64, exclude=None, chunk_elems=1 << 22):
    """(d [q, k] float32, sphere [q, k] int32): the first k of W(i) = {reportable spheres with d <= r_i} of each ball in
    ascending d, then caller index, (+inf, -1) after them.  exclude: [q] caller indices (or -1) left out of W(i)."""
    s = np.asarray(spheres, F32).reshape(-1, 7)
    b = np.asarray(balls, F32).reshape(-1, 4)
    n, q = len(s), len(b)
    ok, valid = sphere_ok(s), ball_ok(b)
    d_out = np.full((q, k), np.inf, F32)
    s_out = np.full((q, k), -1, np.int32)
    step = max(1, chunk_elems // max(n, 1))
    for a in range(0, q, step):
        bb = b[a:a + step]
        d = distances(s, bb[:, :3])
        with np.errstate(invalid="ignore"):
            w = (d <= bb[:, 3:4]) & ok[None, :] & valid[a:a + step, None]
        if exclude is not None:
            ex = np.asarray(exclude)[a:a + step]
            rows = np.flatnonzero(ex >= 0)
            w[rows, ex[rows]] = False
        if w.shape[1] > k:   # only the members up to the k-th smallest d of W(i) (ties included) can be among its first k
            with np.errstate(invalid="ignore"):
                thr = np.partition(np.where(w, d, np.nan), k - 1, axis=1)[:, k - 1:k]   # NaN sorts last: |W(i)| < k
                w &= (d <= thr) | np.isnan(thr)
        rows, cols = np.nonzero(w)
        dv = d[rows, cols]
        order = np.lexsort((cols, dv, rows))          # by ball, then d, then caller index
        rows, cols, dv = rows[order], cols[order], dv[order]
        rank = np.arange(len(rows)) - np.searchsorted(rows, rows, "left")
        keep = rank < k
        d_out[a + rows[keep], rank[keep]] = dv[keep]
        s_out[a + rows[keep], rank[keep]] = cols[keep]
    return d_out, s_out


def assert_same(got, want, what):
    """(d, sphere) equal bit for bit"""
    gd, gs = (np.asarray(x) for x in got)
    wd, ws = (np.asarray(x) for x in want)
    assert gd.shape == wd.shape and gs.shape == ws.shape, (what, gd.shape, wd.shape)
    kk = wd.shape[-1]
    bad = np.flatnonzero(((gd.view(np.int32) != wd.view(np.int32)) | (gs != ws)).reshape(-1, kk).any(-1))
    assert bad.size == 0, (f"{what}: {bad.size} rows of records differ, first {bad[0]}: "
                           f"{list(zip(gd.reshape(-1, kk)[bad[0]], gs.reshape(-1, kk)[bad[0]]))} != "
                           f"{list(zip(wd.reshape(-1, kk)[bad[0]], ws.reshape(-1, kk)[bad[0]]))}")


def first_k(want, k):
    return want[0][..., :k], want[1][..., :k]


def drop_self(got, own):
    """The header's neighbour-graph recipe: from k + 1 records per ball, drop the record of sphere own[i], or the last
    record when own[i] is absent; returns k records per ball"""
    d, s = (np.asarray(x) for x in got)
    q, k1 = s.shape
    hit = s == np.asarray(own)[:, None]
    drop = np.where(hit.any(1), hit.argmax(1), k1 - 1)
    keep = np.ones((q, k1), bool)
    keep[np.arange(q), drop] = False
    return d[keep].reshape(q, k1 - 1), s[keep].reshape(q, k1 - 1)


# ------------------------------------------------------------------------------------------ scenes and balls


def copies_scene(seed=3, groups=60, filler=2000):
    """Groups of 1..24 coincident copies with different radii, scattered through the caller's array, and random filler"""
    rng = np.random.default_rng(seed)
    rows = []
    for g in range(groups):
        c = rng.uniform(-100, 100, 3)
        for _ in range(int(rng.integers(1, 25))):
            rows.append([*c, 0.5, 0.5, 0.5, rng.choice([0.0, 0.5, 1.0, 1.0, 2.0, 4.0])])
    f = np.zeros((filler, 7))
    f[:, :3] = rng.uniform(-100, 100, (filler, 3))
    f[:, 6] = rng.uniform(0.1, 3, filler)
    s = np.concatenate([np.array(rows), f])
    return np.ascontiguousarray(s[rng.permutation(len(s))], F32)


def scene_named(name):
    """(spheres, cam7) of a test scene"""
    if name == "copies":
        return copies_scene(), np.float32([0, 0, 300, 0, 0, 0, 40])
    return TP.scene_named(name)


def nearest_balls(spheres, n_random, seed):
    """Balls of every kind: own centres (up to 1000) unbounded, random points in and around the scene unbounded and with
    finite r from 0 to beyond the scene, points on sphere surfaces, points far outside (unbounded, and with an r that
    reaches nothing), and invalid balls (NaN / inf centre, r NaN / -inf / < 0) between them; r = -0.0 is valid"""
    rng = np.random.default_rng(seed)
    s = np.asarray(spheres, F32)
    mid, ext = TP.scene_extent(s)
    ok = np.flatnonzero(sphere_ok(s))
    own = s[rng.permutation(len(s))[:1000]][:, [0, 1, 2, 6]].copy()
    own[:, 3] = np.inf
    pts = np.empty((n_random, 4))
    pts[:, :3] = mid + rng.uniform(-0.6, 0.6, (n_random, 3)) * ext
    pts[:, 3] = np.inf
    half = n_random // 2
    pts[half:, 3] = ext * rng.uniform(0, 1, n_random - half) ** 4
    pts[half:half + 8, 3] = 0.0
    pts[half + 8, 3] = -0.0
    j = ok[rng.integers(0, len(ok), 200)] if len(ok) else np.zeros(0, np.int64)
    dirs = rng.standard_normal((len(j), 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    on = np.empty((len(j), 4))
    on[:, :3] = s[j, :3].astype(np.float64) + dirs * np.abs(s[j, 6:7]).astype(np.float64)
    on[:, 3] = np.inf
    far = np.empty((64, 4))
    far[:, :3] = mid + rng.standard_normal((64, 3)) * 1e4 * ext
    far[:32, 3] = np.inf
    far[32:, 3] = rng.uniform(0, ext, 32)
    bad = np.tile(pts[:8], (1, 1))
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3, 3] = np.nan, np.inf, -np.inf, -1.0
    bad[4, 3], bad[5, 3], bad[6, 3], bad[7, 3] = np.nan, -np.inf, -1e-30, np.nan
    with np.errstate(over="ignore"):                         # far points of a scene near the f32 limit become inf
        balls = np.concatenate([own, pts, on, far, bad]).astype(F32)
    perm = rng.permutation(len(balls))
    return np.ascontiguousarray(balls[perm], F32)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_nearest(ctx, prepared, balls, k):
    out = ctx.query_nearest(prepared, cuda(balls), k)
    return out["d"].cpu().numpy(), out["sphere"].cpu().numpy()


# ------------------------------------------------------------------------------------------ CPU


def test_oracle_against_kdtree_on_equal_radii():
    """With one radius for every sphere, the k nearest by d are the k nearest centres: scipy's float64 k-d tree agrees
    wherever the k-th and (k+1)-th distances are apart"""
    spatial = pytest.importorskip("scipy.spatial")
    rng = np.random.default_rng(31)
    for rho in (0.0, 0.75):
        s = np.zeros((3000, 7), F32)
        s[:, :3] = rng.uniform(-50, 50, (3000, 3))
        s[:, 6] = rho
        pts = np.empty((400, 4), F32)
        pts[:, :3] = rng.uniform(-70, 70, (400, 3))
        pts[:, 3] = np.inf
        tree = spatial.cKDTree(s[:, :3].astype(np.float64))
        for k in (1, 8, 64):
            d, sp = brute(s, pts, k)
            dist, idx = tree.query(pts[:, :3].astype(np.float64), k + 1)
            dist, idx = dist.reshape(len(pts), -1), idx.reshape(len(pts), -1)
            gaps = np.diff(dist, axis=1)
            clear = (gaps > 1e-4).all(1)                         # f32 errors of d are ~1e-5 here
            assert clear.sum() > 200
            assert np.array_equal(sp[clear], idx[clear, :k])
            assert np.allclose(d[clear], dist[clear, :k] - rho, rtol=0, atol=1e-4)


def test_oracle_orders_pads_and_reports_overflow():
    rng = np.random.default_rng(32)
    s = np.zeros((300, 7), F32)
    s[:, :3] = rng.integers(-3, 4, (300, 3))                 # many equal distances: ties broken by caller index
    s[:, 6] = 0.5
    s[:4, :3] = [[3e38, 3e38, 0], [-3e38, 0, 3e38], [3e38, -3e38, 3e38], [0, 3e38, -3e38]]   # d overflows to +inf
    s[4, 6] = np.nan                                          # never reported
    pts = np.zeros((60, 4), F32)
    pts[:, :3] = rng.integers(-3, 4, (60, 3))
    pts[:, 3] = np.inf
    pts[50:, 3] = rng.uniform(0, 3, 10)
    pts[59] = [0, 0, 0, np.nan]
    d, sp = brute(s, pts, 64)
    cnt = (sp >= 0).sum(1)
    for i in range(60):
        key = list(zip(d[i, :cnt[i]], sp[i, :cnt[i]]))
        assert key == sorted(key)
        assert (d[i, cnt[i]:] == np.inf).all() and (sp[i, cnt[i]:] == -1).all()
    # all 299 reportable spheres are within an unbounded ball: 64 records, none of them the NaN sphere
    assert (cnt[:50] == 64).all() and not (sp == 4).any() and cnt[59] == 0
    # at k = 300 the overflowing spheres are the last records, d = +inf with sphere >= 0, in caller order
    d3, s3 = brute(s, pts[:1], 300)
    assert list(s3[0, 295:299]) == [0, 1, 2, 3] and (d3[0, 295:299] == np.inf).all() and s3[0, 299] == -1
    # an exclusion drops one sphere and moves the rest up
    de, se = brute(s, pts[:50], 63, exclude=sp[:50, 0])
    assert np.array_equal(se, sp[:50, 1:]) and np.array_equal(de.view(np.int32), d[:50, 1:].view(np.int32))
    # the recipe of the header on the oracle itself: k + 1 records, dropped as drop_self does, are the exclusion's first k
    own = np.arange(50, 100)
    pts_own = np.concatenate([s[own, :3], np.full((50, 1), np.inf, F32)], 1)
    assert_same(drop_self(brute(s, pts_own, 9), own), brute(s, pts_own, 8, exclude=own), "recipe on the oracle")
    # chunking does not change the answer
    for part, whole in zip(brute(s, pts, 64, chunk_elems=300), (d, sp)):
        assert np.array_equal(part.view(np.int32), whole.view(np.int32))


def test_argument_checks_without_a_gpu():
    torch = pytest.importorskip("torch")
    for k in (0, -1, 65, 1.5, True, "8", None):
        with pytest.raises(ValueError):
            RB.nearest_k(k)
    assert [RB.nearest_k(k) for k in (1, 64, np.int64(8))] == [1, 64, 8]
    for bad in (torch.zeros((5, 3)), torch.zeros((5, 4)), np.zeros((5, 3), F32), torch.zeros((5, 7)),
                torch.zeros((5, 2)), torch.zeros((5, 3), dtype=torch.float64), torch.zeros((2, 5, 3)), None):
        with pytest.raises(ValueError):
            RB.nearest_points(0, bad)
    for bad in (torch.zeros((2, 5, 3)), torch.zeros((5, 3)), torch.zeros((2, 5, 5))):
        with pytest.raises(ValueError):
            RB.nearest_points(0, bad, B=2)


def test_struct_layouts_and_symbols():
    lib = RB.load_library()
    assert C.sizeof(RB.Ball) == lib.ray_b200_ball_size() == 16
    assert C.sizeof(RB.Near) == lib.ray_b200_near_size() == 8
    assert {"ray_b200_query_nearest", "ray_b200_scene_batch_query_nearest"} <= set(RB.declared_symbols())


# ------------------------------------------------------------------------------------------ GPU


@pytest.fixture(scope="module")
def ctx():
    c = RB.Context(device=0)
    yield c
    c.close()


def prepare(ctx, spheres, cam=None):
    cam = np.float32([0, 0, 60, 0, 0, 0, 40]) if cam is None else cam
    return ctx.prepare_scene_device(64, 64, cuda(np.asarray(spheres, F32)), cam)


def check_ks(ctx, pr, s, balls, what, ks=KS):
    want = brute(s, balls, 64)
    for k in ks:
        assert_same(gpu_nearest(ctx, pr, balls, k), first_k(want, k), f"{what} k={k}")
    return want


def check_self_recipe(ctx, pr, s, what, ks=(1, 8, 63), limit=1500, seed=0):
    """Every reportable sphere's own centre (up to `limit` of them) at k + 1, unbounded: the records without the sphere
    itself are the first k of W minus {i}"""
    ok = np.flatnonzero(sphere_ok(s))
    own = np.random.default_rng(seed).permutation(ok)[:limit]
    balls = np.concatenate([s[own, :3], np.full((len(own), 1), np.inf, F32)], 1)
    for k in ks:
        got = drop_self(gpu_nearest(ctx, pr, balls, k + 1), own)
        assert_same(got, brute(s, balls, k, exclude=own), f"{what}: own centres at k+1={k + 1}")


SCENES = ["rgbbox", "irreg", "random65536", "ranges", "comb", "top", "ties", "facing", "copies"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_scenes_against_brute_force(ctx, name):
    s, cam = scene_named(name)
    pr = prepare(ctx, s, cam)
    balls = nearest_balls(s, 300 if len(s) > 20000 else 1500, seed=len(s))
    launches = ctx.launch_count()
    plan = ctx.last_plan()
    want = check_ks(ctx, pr, s, balls, name)
    stale = pr.info()["stale_nodes"]
    assert ctx.launch_count() - launches == len(KS) * (3 if stale else 1)
    assert ctx.last_plan() == plan
    n_ok = int(sphere_ok(s).sum())
    unbounded = ball_ok(balls) & (balls[:, 3] == np.inf)
    assert ((want[1][unbounded] >= 0).sum(1) == min(64, n_ok)).all(), "an unbounded ball missed a sphere"
    check_self_recipe(ctx, pr, s, name)
    if name == "rgbbox":
        assert stale > 0
    pr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "random65536", "ranges", "copies"])
def test_finite_r_is_query_spheres(ctx, name):
    """For a finite r the records are query_spheres'; at k = 1 record 0's d is the signed distance of the union"""
    s, cam = scene_named(name)
    pr = prepare(ctx, s, cam)
    balls = nearest_balls(s, 2000, seed=7)
    balls = balls[np.isfinite(balls[:, 3]) | ~ball_ok(balls)]
    for k in (1, 8, 64):
        q = ctx.query_spheres(pr, cuda(balls), k)
        assert_same(gpu_nearest(ctx, pr, balls, k), (q["d"].cpu().numpy(), q["sphere"].cpu().numpy()), f"{name} k={k}")
    pts = nearest_balls(s, 2000, seed=8)
    pts = pts[ball_ok(pts)]
    pts[:, 3] = np.inf
    d1 = gpu_nearest(ctx, pr, pts, 1)[0][:, 0]
    ok = sphere_ok(s)
    with np.errstate(invalid="ignore"):
        sdf = distances(s[ok], pts[:, :3]).min(1)
    assert np.array_equal(d1.view(np.int32), sdf.view(np.int32)), f"{name}: the signed distance of the union"
    pr.free()


@pytest.mark.gpu
def test_no_reportable_sphere(ctx):
    s = np.zeros((40, 7), F32)
    s[:, :3] = np.random.default_rng(1).uniform(-10, 10, (40, 3))
    s[:, 6] = np.nan
    s[::3, 6] = -1.0
    pr = prepare(ctx, s)
    pts = np.zeros((100, 4), F32)
    pts[:, :3] = np.random.default_rng(2).uniform(-20, 20, (100, 3))
    pts[:, 3] = np.inf
    d, sp = gpu_nearest(ctx, pr, pts, 8)
    assert (d == np.inf).all() and (sp == -1).all()
    pr.free()


# ------------------------------------------------------------------------------------------ GPU: ties across pruning


@pytest.mark.gpu
def test_lattice_ties(ctx):
    """Spheres on an integer lattice: many at exactly the k-th distance from lattice points, half-integer points and cell
    centres, unbounded and with r at exactly a lattice distance"""
    g = np.stack(np.meshgrid(*[np.arange(16)] * 3, indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(3)
    order = rng.permutation(len(g))
    for rho in (0.5, 0.0):
        s = np.zeros((len(g), 7), F32)
        s[:, :3] = g[order]
        s[:, 6] = rho
        pr = prepare(ctx, s)
        pts = np.concatenate([rng.integers(0, 16, (600, 3)), rng.integers(0, 16, (300, 3)) + 0.5,
                              rng.integers(0, 16, (300, 3)) + [0.5, 0.0, 0.0]]).astype(F32)
        balls = np.concatenate([pts, np.full((len(pts), 1), np.inf, F32)], 1)
        lim = balls.copy()
        lim[:, 3] = np.float32(rng.choice([1.0, np.sqrt(2), np.sqrt(3), 2.0], len(lim))) - F32(rho)
        both = np.concatenate([balls, lim])
        check_ks(ctx, pr, s, both, f"lattice rho={rho}")
        check_self_recipe(ctx, pr, s, f"lattice rho={rho}", ks=(1, 6, 18, 26, 63), limit=800)
        pr.free()


@pytest.mark.gpu
def test_coincident_copies_self_recipe(ctx):
    """Coincident copies with different radii and indices: every sphere's own centre at k + 1 gives the first k of W minus
    {i}, with the copies of i ordered among themselves by radius and index"""
    s = copies_scene(seed=9, groups=120, filler=3000)
    pr = prepare(ctx, s)
    check_self_recipe(ctx, pr, s, "copies", ks=(1, 2, 8, 9, 24, 63), limit=4000, seed=1)
    pr.free()


@pytest.mark.gpu
def test_nested_spheres_negative_dk(ctx):
    """Spheres that all contain the query points, their centres spread over the scene so that they sit in different
    subtrees, and concentric ones: d_k < 0, so the walk prunes with R = 0"""
    rng = np.random.default_rng(4)
    nested = np.zeros((300, 7), F32)
    nested[:, :3] = rng.uniform(-40, 40, (300, 3))
    nested[:, 6] = rng.uniform(150, 250, 300)   # |p - c| <= 60 sqrt(3) < 150
    conc = np.zeros((40, 7), F32)
    conc[:, 6] = rng.uniform(1, 90, 40)
    filler = np.zeros((5000, 7), F32)
    filler[:, :3] = rng.uniform(-1000, 1000, (5000, 3))
    filler[:, 6] = rng.uniform(0.5, 5, 5000)
    s = np.concatenate([nested, conc, filler])
    s = np.ascontiguousarray(s[rng.permutation(len(s))])
    pr = prepare(ctx, s)
    pts = np.zeros((1500, 4), F32)
    pts[:, :3] = rng.uniform(-20, 20, (1500, 3))
    pts[:, 3] = np.inf
    pts[1000:, 3] = rng.uniform(0, 50, 500)
    pts[:50, :3] = 0.0
    want = check_ks(ctx, pr, s, pts, "nested")
    assert (want[0][:1000, 63] < 0).all(), "premise: d_k < 0 at k = 64"
    pr.free()


# ------------------------------------------------------------------------------------------ GPU: magnitudes


@pytest.mark.gpu
def test_far_tiny_huge_and_overflowing_scenes(ctx):
    """Spheres around 1e6 with radii 1e-6 (R small against M), huge spheres, and spheres whose d from the points overflows
    to +inf: with no limit they are still records, sphere >= 0"""
    rng = np.random.default_rng(5)
    far = np.zeros((4000, 7), F32)
    far[:, :3] = F32(1e6) + rng.uniform(-1, 1, (4000, 3)).astype(F32)
    far[:, 6] = F32(1e-6)
    huge = np.zeros((3000, 7), F32)
    huge[:, :3] = rng.uniform(-1e15, 1e15, (3000, 3))
    huge[:, 6] = rng.uniform(1e12, 1e14, 3000)
    huge[:10, 6] = F32(-0.0)
    over = np.zeros((500, 7), F32)
    over[:, :3] = rng.uniform(-3e38, 3e38, (500, 3))
    over[:, 6] = rng.uniform(0, 1e30, 500)
    over[:50, :3] = rng.uniform(-10, 10, (50, 3))
    for name, s in (("1e6", far), ("huge", huge), ("overflow", over)):
        pr = prepare(ctx, s)
        balls = nearest_balls(s, 1500, seed=11)
        # points right next to spheres, at a fraction of a radius and of the spacing
        j = rng.integers(0, len(s), 500)
        near = np.concatenate([s[j, :3] + rng.standard_normal((500, 3)).astype(F32) * (np.abs(s[j, 6:7]) + F32(1e-3)),
                               np.full((500, 1), np.inf, F32)], 1).astype(F32)
        want = check_ks(ctx, pr, s, np.concatenate([balls, near]), name, ks=(1, 8, 9, 64))
        if name == "overflow":
            assert ((want[0] == np.inf) & (want[1] >= 0)).any(), "premise: records at d = +inf"
        check_self_recipe(ctx, pr, s, name, ks=(1, 8))
        pr.free()


# ------------------------------------------------------------------------------------------ GPU: stale boxes, batches


@pytest.mark.gpu
def test_stale_trees_and_updates(ctx):
    """A 2^16 scene queried before and after updates that make its boxes stale and complete again"""
    fresh, cam = RB.host_scene("random", 1 << 16, 3)
    ties = LS.tie_groups(filler=(1 << 16) - 203)[0]
    rg = RB.host_scene("rgbbox")[0]
    pr = prepare(ctx, fresh, cam)
    seen = []
    for step, s in enumerate((fresh, ties, fresh, rg, ties)):
        if step:
            pr.update(cuda(s))
        stale = pr.info()["stale_nodes"]
        seen.append(stale > 0)
        balls = nearest_balls(s, 300, seed=step)
        check_ks(ctx, pr, s, balls, f"update step {step} (stale {stale})", ks=(1, 9, 64))
        check_self_recipe(ctx, pr, s, f"update step {step}", ks=(8,), limit=500)
    assert seen == [False, True, False, True, True], seen
    pr.free()


def batch_members_check(ctx, batch, parts, balls, ks=(1, 8, 9, 64)):
    """Every ball of scene b equals query_nearest on batch.member(b) and the brute force on scene b's records"""
    for k in ks:
        out = ctx.query_scene_batch_nearest(batch, cuda(balls), k)
        got = [x.cpu().numpy() for x in (out["d"], out["sphere"])]
        for b, s in enumerate(parts):
            mem = batch.member(b)
            one = gpu_nearest(ctx, mem, balls[b], k)
            assert_same((got[0][b], got[1][b]), one, f"batch member {b} k={k}")
            assert_same(one, brute(s, balls[b], k), f"batch member {b} k={k} vs brute force")
            mem.free()


@pytest.mark.gpu
def test_uniform_batch(ctx):
    rng = np.random.default_rng(5)   # a mix of members with and without stale boxes
    B, n, m = 24, 64, 48
    s = np.zeros((B, n, 7), F32)
    s[..., :3] = rng.uniform(-20, 20, (B, n, 3))
    s[..., 3:6] = 0.5
    s[..., 6] = rng.uniform(0.5, 4, (B, n))
    stale = [RB.host_lbvh(s[b])["stale_nodes"] for b in range(B)]
    assert any(stale) and not all(stale), stale
    batch = ctx.prepare_scene_batch(64, 64, cuda(s), np.tile(np.float32([0, 0, 60, 0, 0, 0, 40]), (B, 1)))
    balls = np.stack([nearest_balls(s[b], m, seed=b)[:m] for b in range(B)])
    batch_members_check(ctx, batch, list(s), balls)
    # [B, m, 3] points are unbounded balls
    pts = np.ascontiguousarray(balls[..., :3])
    out = ctx.query_scene_batch_nearest(batch, cuda(pts), 5)
    inf_balls = np.concatenate([pts, np.full(pts.shape[:2] + (1,), np.inf, F32)], -1)
    for b in range(B):
        assert_same((out["d"][b].cpu().numpy(), out["sphere"][b].cpu().numpy()), brute(s[b], inf_balls[b], 5), f"points {b}")
    batch.free()


@pytest.mark.gpu
def test_ragged_batch(ctx):
    parts = [RB.host_scene("rgbbox")[0], RB.host_scene("random", 3000, 2)[0], RB.host_scene("random", 2, 1)[0],
             TP.input_range_scene(9, 500), LS.comb_scene(100)[0], copies_scene(4, 20, 100)]
    counts = [len(p) for p in parts]
    cams = np.tile(np.float32([0, 0, 60, 0, 0, 0, 40]), (len(parts), 1))
    batch = ctx.prepare_scene_batch(64, 64, cuda(np.concatenate(parts)), cams, counts=counts)
    m = 200
    balls = np.stack([nearest_balls(p, m, seed=b)[:m] for b, p in enumerate(parts)])
    batch_members_check(ctx, batch, parts, balls)
    parts2 = [parts[1][:17], parts[0], parts[3][:300], parts[2], parts[4], parts[5][:50]]
    batch.update(cuda(np.concatenate(parts2)), counts=[len(p) for p in parts2])
    balls2 = np.stack([nearest_balls(p, m, seed=10 + b)[:m] for b, p in enumerate(parts2)])
    batch_members_check(ctx, batch, parts2, balls2, ks=(9,))
    out = ctx.query_scene_batch_nearest(batch, cuda(np.zeros((len(parts2), 0, 4), F32)), 8)   # m = 0 does nothing
    assert out["d"].shape == (len(parts2), 0, 8)
    batch.free()


# ------------------------------------------------------------------------------------------ GPU: the contract


@pytest.fixture(scope="module")
def env():
    import test_memory_contract as M
    e = M.Env()
    yield e
    e.close()


def _guarded_query(e, pr, balls, k, sentinel, align=16):
    import test_memory_contract as M
    n = len(balls)
    got = M.run_call(e, lambda p: e.ctx.query_nearest_into(p["balls"], n, pr, k, p["near"]), {"near": n * k * 8},
                     ins={"balls": (balls, align)}, sentinel=sentinel, what=f"query_nearest k={k}")
    near = got["near"].view(np.int32).reshape(n, k, 2)
    return near[..., 0].view(F32), near[..., 1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_guarded_outputs(env, name):
    s, cam = scene_named(name)
    pr = prepare(env.ctx, s, cam)
    balls = nearest_balls(s, 500, seed=3)
    want = brute(s, balls, 64)
    for k in (1, 7, 64):
        for sent in (0x00, 0xFF):
            assert_same(_guarded_query(env, pr, balls, k, sent, align=4 if k == 7 else 16), first_k(want, k),
                        f"guarded {name} k={k}")
    pr.free()


@pytest.mark.gpu
def test_poisoned_scratch(env):
    """The complete-box scratch of a stale scene is not trusted: results are the same whatever the pool held"""
    import test_memory_contract as M
    s, cam = scene_named("rgbbox")
    pr = prepare(env.ctx, s, cam)
    balls = nearest_balls(s, 500, seed=4)
    want = brute(s, balls, 8)
    env.driver = M.Driver(0)
    try:
        for pattern in M.PATTERNS:
            env.pattern = pattern
            assert_same(_guarded_query(env, pr, balls, 8, 0x00), want, f"pattern {pattern:#x}")
    finally:
        env.pattern = None
    pr.free()


@pytest.mark.gpu
def test_errors_write_nothing(env):
    import test_memory_contract as M
    s, cam = scene_named("rgbbox")
    pr = prepare(env.ctx, s, cam)
    batch = env.ctx.prepare_scene_batch(64, 64, cuda(np.stack([s[:20], s[20:40]])), np.stack([cam, cam]))
    balls = nearest_balls(s, 64, seed=5)
    n = len(balls)
    lib, h = env.ctx.lib, env.ctx.handle
    calls = {
        "k = 0": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], n, 0, p["near"]),
        "k = -1": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], n, -1, p["near"]),
        "k = 65": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], n, 65, p["near"]),
        "n < 0": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], -1, 8, p["near"]),
        "n > 2^30": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], (1 << 30) + 1, 8, p["near"]),
        "NULL balls": lambda p: lib.ray_b200_query_nearest(h, pr.handle, None, n, 8, p["near"]),
        "NULL near": lambda p: lib.ray_b200_query_nearest(h, pr.handle, p["balls"], n, 8, None),
        "NULL scene": lambda p: lib.ray_b200_query_nearest(h, None, p["balls"], n, 8, p["near"]),
        "NULL batch": lambda p: lib.ray_b200_scene_batch_query_nearest(h, None, p["balls"], n, 8, p["near"]),
        "batch m < 0": lambda p: lib.ray_b200_scene_batch_query_nearest(h, batch.handle, p["balls"], -1, 8, p["near"]),
        "batch B m > 2^30": lambda p: lib.ray_b200_scene_batch_query_nearest(h, batch.handle, p["balls"], (1 << 29) + 1, 8,
                                                                             p["near"]),
        "batch k = 0": lambda p: lib.ray_b200_scene_batch_query_nearest(h, batch.handle, p["balls"], n // 2, 0, p["near"]),
    }
    for what, call in calls.items():
        rcs = []
        got = M.run_call(env, lambda p: rcs.append(call(p)), {"near": n * 8 * 8}, ins={"balls": (balls, 16)}, sentinel=0xFF,
                         what=what)
        assert rcs[0] != 0, what
        assert env.ctx.get_error(), what
        assert (got["near"] == 0xFF).all(), f"{what}: an output was written"
        assert_same(gpu_nearest(env.ctx, pr, balls, 8), brute(s, balls, 8), f"after {what}")   # the context stays usable
    assert lib.ray_b200_query_nearest(h, pr.handle, None, 0, 8, None) == 0                    # n == 0 does nothing
    batch.free()
    pr.free()


@pytest.mark.gpu
def test_stream_order_and_scenes_freed_in_flight():
    """Balls written by a producer on the context's stream are read after it; a scene freed or updated right after a
    query was enqueued still gives that query the old scene's answer"""
    import torch
    s, cam = RB.host_scene("random", 1 << 16, 4)
    s2, _ = RB.host_scene("random", 1 << 16, 5)
    balls = nearest_balls(s, 2000, seed=6)
    want = brute(s, balls, 8)
    with RB.Context(device=0) as c:
        stream = torch.cuda.Stream()
        c.set_stream(stream.cuda_stream)
        for action in ("free", "update"):
            pr = c.prepare_scene_device(64, 64, cuda(s), cam)
            s2_dev = cuda(s2)
            torch.cuda.synchronize()
            src = cuda(balls)
            dst = torch.full_like(src, float("nan"))
            near = torch.empty((len(balls), 8, 2), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(50_000_000)            # the producer is still running when the query is enqueued
                dst.copy_(src)
            c.query_nearest_into(dst.data_ptr(), len(balls), pr, 8, near.data_ptr())
            if action == "free":
                pr.free()
            else:
                pr.update_from_ptr(s2_dev.data_ptr(), len(s2))
            c.sync()
            got = (near[..., 0].cpu().numpy(), near[..., 1].view(torch.int32).cpu().numpy())
            assert_same(got, want, f"producer on the stream, scene {action}d in flight")
            if action == "update":
                assert_same(gpu_nearest(c, pr, balls, 8), brute(s2, balls, 8), "after the update")
                pr.free()
