"""Proximity queries (include/ray_b200.h "proximity queries"): the spheres within a radius of each ball, nearest first.

The oracle is a brute force over every sphere of a scene in numpy float32, with the header's operation order: numpy's
float32 ufuncs round every operation to nearest and np.sqrt on float32 is correctly rounded, as the kernel's __fsqrt_rn
is.  Every GPU output must equal it bit for bit: counts, the bits of d, sphere indices, and the padding records.

- CPU: the oracle against a float64 computation away from the boundary, its ordering and padding, and the Python argument
  checks.
- GPU: built-in, random, limit and input-range scenes with self-overlap balls, random points with r from 0 to beyond the
  scene, far and invalid balls at k = 0, 1, 4, 8 and 64; >= 10^4 (ball, sphere) pairs at r = d and nextafter(d, -inf);
  scenes with stale boxes, before and after updates that change stale_nodes, and a float64 k-d tree as an independent
  check; uniform and ragged scene batches against their members; guarded outputs, errors, stream order and freeing or
  updating a scene with a query in flight.
"""
import ctypes as C

import numpy as np
import pytest

import limit_scenes as LS
import raytracers_b200 as RB

KS = (0, 1, 4, 8, 64)
F32 = np.float32

# ------------------------------------------------------------------------------------------ the oracle


def sphere_ok(spheres):
    """Which spheres can be reported: finite centre and radius, radius >= 0 (-0.0 included)"""
    s = np.asarray(spheres, F32)
    with np.errstate(invalid="ignore"):
        return np.isfinite(s[:, :3]).all(1) & np.isfinite(s[:, 6]) & (s[:, 6] >= 0)


def ball_ok(balls):
    b = np.asarray(balls, F32)
    with np.errstate(invalid="ignore"):
        return np.isfinite(b[:, :3]).all(1) & np.isfinite(b[:, 3]) & (b[:, 3] >= 0)


def distances(spheres, centres):
    """d[q, j] = sqrtf((dx*dx + dy*dy) + dz*dz) - rho in float32, dx = p.x - c.x, for every ball centre and sphere"""
    s = np.asarray(spheres, F32)
    c = np.asarray(centres, F32)
    with np.errstate(all="ignore"):
        dx = s[None, :, 0] - c[:, None, 0]
        dy = s[None, :, 1] - c[:, None, 1]
        dz = s[None, :, 2] - c[:, None, 2]
        return np.sqrt((dx * dx + dy * dy) + dz * dz) - s[None, :, 6]


def brute(spheres, balls, k=64, chunk_elems=1 << 22):
    """(d [q, k] float32, sphere [q, k] int32, count [q] int32) of a brute force over every sphere, chunked over balls"""
    s = np.asarray(spheres, F32).reshape(-1, 7)
    b = np.asarray(balls, F32).reshape(-1, 4)
    n, q = len(s), len(b)
    ok, valid = sphere_ok(s), ball_ok(b)
    d_out = np.full((q, k), np.inf, F32)
    s_out = np.full((q, k), -1, np.int32)
    count = np.zeros(q, np.int32)
    step = max(1, chunk_elems // max(n, 1))
    for a in range(0, q, step):
        bb = b[a:a + step]
        d = distances(s, bb[:, :3])
        with np.errstate(invalid="ignore"):
            w = (d <= bb[:, 3:4]) & ok[None, :] & valid[a:a + step, None]
        count[a:a + len(bb)] = w.sum(1)
        if k:
            rows, cols = np.nonzero(w)
            dv = d[rows, cols]
            order = np.lexsort((cols, dv, rows))          # by ball, then d, then caller index
            rows, cols, dv = rows[order], cols[order], dv[order]
            rank = np.arange(len(rows)) - np.searchsorted(rows, rows, "left")
            keep = rank < k
            d_out[a + rows[keep], rank[keep]] = dv[keep]
            s_out[a + rows[keep], rank[keep]] = cols[keep]
    return d_out, s_out, count


def assert_same(got, want, what):
    """(d, sphere, count) equal bit for bit"""
    gd, gs, gc = (np.asarray(x) for x in got)
    wd, ws, wc = (np.asarray(x) for x in want)
    assert gc.shape == wc.shape and gd.shape == wd.shape, (what, gd.shape, wd.shape)
    bad_c = np.flatnonzero(gc != wc)
    assert bad_c.size == 0, f"{what}: {bad_c.size} counts differ, first ball {bad_c[0]}: {gc[bad_c[0]]} != {wc[bad_c[0]]}"
    bad = np.flatnonzero(((gd.view(np.int32) != wd.view(np.int32)) | (gs != ws)).any(-1).reshape(-1))
    assert bad.size == 0, (f"{what}: {bad.size} rows of records differ, first {bad[0]}: "
                           f"{list(zip(gd.reshape(-1, wd.shape[-1])[bad[0]], gs.reshape(-1, wd.shape[-1])[bad[0]]))} != "
                           f"{list(zip(wd.reshape(-1, wd.shape[-1])[bad[0]], ws.reshape(-1, wd.shape[-1])[bad[0]]))}")


def pair_d(rows, centres):
    """d of sphere rows[i] from centres[i], elementwise, in the header's order"""
    s = np.asarray(rows, F32)
    c = np.asarray(centres, F32)
    with np.errstate(all="ignore"):
        dx, dy, dz = s[:, 0] - c[:, 0], s[:, 1] - c[:, 1], s[:, 2] - c[:, 2]
        return np.sqrt((dx * dx + dy * dy) + dz * dz) - s[:, 6]


def first_k(want, k):
    d, s, c = want
    return d[..., :k], s[..., :k], c


# ------------------------------------------------------------------------------------------ scenes and balls


def input_range_scene(seed=7, n=3000):
    """Random spheres with the inputs outside the built-in ranges: NaN and infinite centre components and radii, negative
    radii, radius -0.0 and +0.0, coincident copies, and spheres far out (1e6) and tiny (1e-6)"""
    rng = np.random.default_rng(seed)
    s = np.zeros((n, 7), F32)
    s[:, :3] = rng.uniform(-100, 100, (n, 3))
    s[:, 3:6] = rng.uniform(0.1, 1, (n, 3))
    s[:, 6] = rng.uniform(0.1, 8, n)
    idx = rng.permutation(n)
    s[idx[0:20], 6] = np.nan
    s[idx[20:40], 6] = -rng.uniform(0.1, 5, 20)
    s[idx[40:50], 6] = np.inf
    s[idx[50:60], rng.integers(0, 3, 10)] = np.nan
    s[idx[60:70], 0] = np.inf
    s[idx[70:80], 1] = -np.inf
    s[idx[80:100], 6] = F32(-0.0)
    s[idx[100:120], 6] = F32(0.0)
    s[idx[120:160]] = s[idx[160]]                       # 40 coincident copies of one sphere
    s[idx[160:200], :3] += F32(1e6)
    s[idx[200:240], 6] = F32(1e-6)
    return np.ascontiguousarray(s)


def scene_named(name):
    """(spheres, cam7) of a test scene"""
    if name in ("rgbbox", "irreg"):
        return RB.host_scene(name)
    if name.startswith("random"):
        return RB.host_scene("random", int(name[6:]), 3)
    if name == "comb":
        return LS.comb_scene(300)[0], LS.COMB_CAM
    if name == "top":
        s, cam, _ = LS.top_of_index_scene(4096)
        return s, cam
    if name == "ties":
        return LS.tie_groups(filler=2000)[0], LS.TIE_CAM
    if name == "facing":
        return LS.facing_spheres(10.0, 1e-3), LS.FACING_CAM
    if name == "ranges":
        return input_range_scene(), np.float32([0, 0, 400, 0, 0, 0, 40])
    raise KeyError(name)


def scene_extent(spheres):
    s = np.asarray(spheres, F32)
    ok = sphere_ok(s)
    c = s[ok, :3].astype(np.float64)
    if not len(c):
        return np.zeros(3), 1.0
    lo, hi = c.min(0), c.max(0)
    return (lo + hi) / 2, float(np.linalg.norm(hi - lo) + 2 * s[ok, 6].max() + 1)


def query_balls(spheres, n_random, seed):
    """Self-overlap balls of every sphere (up to 2000), random points with r from 0 up to beyond the scene (a few with
    every sphere within), points far outside, and invalid balls (NaN / inf centre, r < 0, r NaN / inf) between them"""
    rng = np.random.default_rng(seed)
    s = np.asarray(spheres, F32)
    mid, ext = scene_extent(s)
    own = s[rng.permutation(len(s))[:2000]][:, [0, 1, 2, 6]]
    pts = np.empty((n_random, 4))
    pts[:, :3] = mid + rng.uniform(-0.6, 0.6, (n_random, 3)) * ext
    pts[:, 3] = ext * rng.uniform(0, 1, n_random) ** 4
    pts[:8, 3] = 0.0
    pts[8:11, 3] = 2 * ext                                   # every sphere within
    far = np.empty((64, 4))
    far[:, :3] = mid + rng.standard_normal((64, 3)) * 1e4 * ext
    far[:, 3] = rng.uniform(0, ext, 64)
    bad = np.tile(pts[:8], (1, 1))
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3, 3] = np.nan, np.inf, -np.inf, -1.0
    bad[4, 3], bad[5, 3], bad[6, 3], bad[7, 3] = np.nan, np.inf, -np.inf, -1e-30
    balls = np.concatenate([own, pts.astype(F32), far.astype(F32), bad.astype(F32)])
    balls = balls[rng.permutation(len(balls))]               # invalid balls between valid ones
    return np.ascontiguousarray(balls, F32)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_query(ctx, prepared, balls, k):
    out = ctx.query_spheres(prepared, cuda(balls), k)
    return out["d"].cpu().numpy(), out["sphere"].cpu().numpy(), out["count"].cpu().numpy()


def check_all_ks(ctx, prepared, spheres, balls, what, ks=KS):
    want = brute(spheres, balls, 64)
    for k in ks:
        assert_same(gpu_query(ctx, prepared, balls, k), first_k(want, k), f"{what} k={k}")
    return want


# ------------------------------------------------------------------------------------------ CPU


def test_oracle_against_float64_away_from_the_boundary():
    rng = np.random.default_rng(11)
    s = np.zeros((700, 7), F32)
    s[:, :3] = rng.uniform(-50, 50, (700, 3))
    s[:, 6] = rng.uniform(0.1, 4, 700)
    s[:5, 6] = F32(-0.0)
    balls = np.zeros((300, 4), F32)
    balls[:, :3] = rng.uniform(-60, 60, (300, 3))
    balls[:, 3] = rng.uniform(0, 30, 300)
    d, sp, cnt = brute(s, balls, 64)
    d64 = np.linalg.norm(s[None, :, :3].astype(np.float64) - balls[:, None, :3].astype(np.float64), axis=2) - s[None, :, 6]
    r = balls[:, 3:4].astype(np.float64)
    clear = np.abs(d64 - r) > 1e-4 * (np.abs(r) + 100)
    assert clear.mean() > 0.99
    rows = clear.all(1)                                     # balls with no sphere near their boundary
    assert rows.sum() > 100
    assert np.array_equal(cnt[rows], (d64 <= r).sum(1)[rows])
    for i in np.flatnonzero(rows & (cnt <= 64)):
        want = np.flatnonzero(d64[i] <= r[i])
        want = want[np.lexsort((want, d64[i, want]))]
        assert set(sp[i, :cnt[i]]) == set(want)
        assert np.allclose(d[i, :cnt[i]], d64[i, sp[i, :cnt[i]]], rtol=0, atol=1e-4)


def test_oracle_orders_and_pads():
    rng = np.random.default_rng(12)
    s = np.zeros((200, 7), F32)
    s[:, :3] = rng.integers(-3, 4, (200, 3))                 # many equal distances: ties broken by caller index
    s[:, 6] = 0.5
    balls = np.zeros((50, 4), F32)
    balls[:, :3] = rng.integers(-3, 4, (50, 3))
    balls[:, 3] = rng.uniform(0, 3, 50)
    d, sp, cnt = brute(s, balls, 64)
    for i in range(50):
        c = min(cnt[i], 64)
        key = list(zip(d[i, :c], sp[i, :c]))
        assert key == sorted(key)
        assert (d[i, c:] == np.inf).all() and (sp[i, c:] == -1).all()
        assert not np.signbit(d[i, :c][d[i, :c] == 0]).any()   # never -0.0
    # chunking does not change the answer
    for part, whole in zip(brute(s, balls, 64, chunk_elems=300), (d, sp, cnt)):
        assert np.array_equal(part.view(np.int32) if part.dtype == F32 else part,
                              whole.view(np.int32) if whole.dtype == F32 else whole)


def test_oracle_reports_only_valid_spheres_and_balls():
    s = input_range_scene(3, 500)
    balls = np.array([[0, 0, 0, 1e4], [np.nan, 0, 0, 1], [0, 0, 0, -1], [0, 0, 0, np.inf], [0, 0, 0, F32(-0.0)]], F32)
    d, sp, cnt = brute(s, balls, 64)
    ok = sphere_ok(s)
    assert not ok.all() and ok[np.isnan(s[:, 6]) | (s[:, 6] < 0) | ~np.isfinite(s[:, :3]).all(1)].sum() == 0
    assert ok[s[:, 6] == 0].all()                           # +0.0 and -0.0 are point spheres
    with np.errstate(invalid="ignore"):
        assert cnt[0] == (ok & (distances(s, balls[:1, :3])[0] <= 1e4)).sum() > 300
    assert set(sp[0][sp[0] >= 0]) <= set(np.flatnonzero(ok))
    assert (cnt[1:4] == 0).all() and (sp[1:4] == -1).all()
    assert cnt[4] == 0 and ball_ok(balls[4:])[0]            # r = -0.0 is valid; no sphere centre sits at the origin


def test_argument_checks_without_a_gpu():
    torch = pytest.importorskip("torch")
    for k in (-1, 65, 1.5, True, "8", None):
        with pytest.raises(ValueError):
            RB.proximity_k(k)
    assert [RB.proximity_k(k) for k in (0, 1, 64, np.int64(8))] == [0, 1, 64, 8]
    cpu = torch.zeros((5, 4), dtype=torch.float32)
    for bad in (cpu, np.zeros((5, 4), F32), torch.zeros((5, 7)), torch.zeros((5, 4), dtype=torch.float64), None):
        with pytest.raises(ValueError):
            RB.proximity_balls(0, bad)
    with pytest.raises(ValueError):
        RB.proximity_balls(0, torch.zeros((2, 5, 4)), B=2)    # a host tensor


def test_struct_layouts_match_the_library():
    lib = RB.load_library()
    assert C.sizeof(RB.Ball) == lib.ray_b200_ball_size() == 16
    assert C.sizeof(RB.Near) == lib.ray_b200_near_size() == 8
    assert {"ray_b200_query_spheres", "ray_b200_scene_batch_query_spheres"} <= set(RB.declared_symbols())


# ------------------------------------------------------------------------------------------ GPU


@pytest.fixture(scope="module")
def ctx():
    c = RB.Context(device=0)
    yield c
    c.close()


def prepare(ctx, spheres, cam):
    return ctx.prepare_scene_device(64, 64, cuda(np.asarray(spheres, F32)), cam)


SCENES = ["rgbbox", "irreg", "random1024", "random65536", "comb", "top", "ties", "facing", "ranges"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_scenes_against_brute_force(ctx, name):
    s, cam = scene_named(name)
    pr = prepare(ctx, s, cam)
    n_random = 300 if len(s) > 20000 else 1500
    balls = query_balls(s, n_random, seed=len(s))
    launches = ctx.launch_count()
    plan = ctx.last_plan()
    want = check_all_ks(ctx, pr, s, balls, name)
    stale = pr.info()["stale_nodes"]
    assert ctx.launch_count() - launches == len(KS) * (3 if stale else 1)
    assert ctx.last_plan() == plan
    assert (want[2] > 64).any() or len(s) <= 64, "no count above the largest k"
    if name == "rgbbox":
        assert stale > 0


@pytest.mark.gpu
def test_boundary_pairs(ctx):
    """r = the pair's own f32 d counts the sphere, r = nextafter(d, -inf) does not, for >= 10^4 pairs per scene: around
    1e6 with radii 1e-6, huge spheres, and a scene with stale boxes"""
    rng = np.random.default_rng(21)
    scenes = []
    far = np.zeros((3000, 7), F32)
    far[:, :3] = F32(1e6) + rng.uniform(-1, 1, (3000, 3)).astype(F32)
    far[:, 6] = F32(1e-6)
    scenes.append(("1e6", far))
    huge = np.zeros((2000, 7), F32)
    huge[:, :3] = rng.uniform(-1e15, 1e15, (2000, 3))
    huge[:, 6] = rng.uniform(1e12, 1e14, 2000)
    huge[:10, 6] = F32(-0.0)
    scenes.append(("huge", huge))
    scenes.append(("rgbbox", RB.host_scene("rgbbox")[0]))
    scenes.append(("ranges", input_range_scene(5, 2000)))
    total = 0
    for name, s in scenes:
        ok = np.flatnonzero(sphere_ok(s))
        j = ok[rng.integers(0, len(ok), 6000)]
        mid, ext = scene_extent(s)
        dirs = rng.standard_normal((len(j), 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        gap = np.abs(s[j, 6]).astype(np.float64) * rng.uniform(0, 3, len(j)) + rng.uniform(0, 1e-3, len(j)) * ext
        c = (s[j, :3].astype(np.float64) + dirs * (np.abs(s[j, 6])[:, None] + gap[:, None])).astype(F32)
        d = pair_d(s[j], c)
        use = np.isfinite(d) & (d >= 0)
        c, d, j = c[use], d[use], j[use]
        below = np.nextafter(d, F32(-np.inf))
        keep = below >= 0
        balls = np.concatenate([np.concatenate([c, d[:, None]], 1), np.concatenate([c[keep], below[keep, None]], 1)]).astype(F32)
        pr = prepare(ctx, s, np.float32([0, 0, 1, 0, 0, 0, 40]))
        want = brute(s, balls, 4)
        got = gpu_query(ctx, pr, balls, 4)
        assert_same(got, want, f"boundary {name}")
        # the premise: the pair's sphere is within at r = d and not at the next float below
        assert (pair_d(s[j], c) <= d).all() and not (pair_d(s[j[keep]], c[keep]) <= below[keep]).any()
        assert (want[2][:len(d)] >= 1).all()
        total += len(d) + int(keep.sum())
        pr.free()
    assert total >= 3 * 10 ** 4


@pytest.mark.gpu
def test_stale_trees_and_updates(ctx):
    """A 2^16 scene queried before and after updates that make its boxes stale and complete again, and an independent
    float64 k-d tree agreeing with the sphere sets away from the boundary"""
    spatial = pytest.importorskip("scipy.spatial")
    fresh, cam = RB.host_scene("random", 1 << 16, 3)
    ties = LS.tie_groups(filler=(1 << 16) - 203)[0]
    assert len(ties) == 1 << 16
    pr = prepare(ctx, fresh, cam)
    seen = []
    for step, s in enumerate((fresh, ties, fresh, ties)):
        if step:
            pr.update(cuda(s))
        stale = pr.info()["stale_nodes"]
        seen.append(stale > 0)
        balls = query_balls(s, 300, seed=step)
        want = check_all_ks(ctx, pr, s, balls, f"update step {step} (stale {stale})", ks=(0, 8, 64))
        if step == 1:
            tree = spatial.cKDTree(s[:, :3].astype(np.float64))
            rho_max = float(s[:, 6].max())
            for i in np.flatnonzero(ball_ok(balls) & (want[2] <= 64))[:200]:
                c, r = balls[i, :3].astype(np.float64), float(balls[i, 3])
                cand = np.array(tree.query_ball_point(c, r + rho_max + 1e-3), np.int64)
                d64 = np.linalg.norm(s[cand, :3].astype(np.float64) - c, axis=1) - s[cand, 6]
                near_edge = np.abs(d64 - r) <= 1e-5 * (abs(r) + s[cand, 6] + np.abs(d64) + 1e-30)
                inside = set(cand[(d64 <= r) & ~near_edge])
                maybe = set(cand[near_edge])
                got = set(want[1][i][want[1][i] >= 0])
                assert inside <= got <= inside | maybe, i
    assert seen == [False, True, False, True], seen
    pr.free()


def batch_members_check(ctx, batch, parts, balls, ks=(0, 1, 8, 64)):
    """Every ball of scene b equals query_spheres on batch.member(b) and the brute force on scene b's records"""
    for k in ks:
        out = ctx.query_scene_batch_spheres(batch, cuda(balls), k)
        got = [x.cpu().numpy() for x in (out["d"], out["sphere"], out["count"])]
        for b, s in enumerate(parts):
            mem = batch.member(b)
            one = gpu_query(ctx, mem, balls[b], k)
            assert_same((got[0][b], got[1][b], got[2][b]), one, f"batch member {b} k={k}")
            assert_same(one, brute(s, balls[b], k), f"batch member {b} k={k} vs brute force")
            mem.free()


@pytest.mark.gpu
def test_uniform_batch(ctx):
    rng = np.random.default_rng(5)
    B, n, m = 24, 64, 48
    s = np.zeros((B, n, 7), F32)
    s[..., :3] = rng.uniform(-20, 20, (B, n, 3))
    s[..., 3:6] = 0.5
    s[..., 6] = rng.uniform(0.5, 4, (B, n))
    stale = [RB.host_lbvh(s[b])["stale_nodes"] for b in range(B)]
    assert any(stale) and not all(stale), stale
    batch = ctx.prepare_scene_batch(64, 64, cuda(s), np.tile(np.float32([0, 0, 60, 0, 0, 0, 40]), (B, 1)))
    balls = np.stack([query_balls(s[b], m, seed=b)[:m] for b in range(B)])
    batch_members_check(ctx, batch, list(s), balls)
    batch.free()


@pytest.mark.gpu
def test_ragged_batch(ctx):
    parts = [RB.host_scene("rgbbox")[0], RB.host_scene("random", 3000, 2)[0], RB.host_scene("random", 2, 1)[0],
             input_range_scene(9, 500), LS.comb_scene(100)[0]]
    counts = [len(p) for p in parts]
    cams = np.tile(np.float32([0, 0, 60, 0, 0, 0, 40]), (len(parts), 1))
    batch = ctx.prepare_scene_batch(64, 64, cuda(np.concatenate(parts)), cams, counts=counts)
    m = 200
    balls = np.stack([query_balls(p, m, seed=b)[:m] for b, p in enumerate(parts)])
    batch_members_check(ctx, batch, parts, balls)
    # updated to other counts: the answers follow the new members
    parts2 = [parts[1][:17], parts[0], parts[3][:300], parts[2], parts[4]]
    batch.update(cuda(np.concatenate(parts2)), counts=[len(p) for p in parts2])
    balls2 = np.stack([query_balls(p, m, seed=10 + b)[:m] for b, p in enumerate(parts2)])
    batch_members_check(ctx, batch, parts2, balls2, ks=(8,))
    # m = 0 does nothing
    out = ctx.query_scene_batch_spheres(batch, cuda(np.zeros((len(parts2), 0, 4), F32)), 8)
    assert out["count"].shape == (len(parts2), 0)
    batch.free()


# ------------------------------------------------------------------------------------------ GPU: the contract


@pytest.fixture(scope="module")
def env():
    import test_memory_contract as M
    e = M.Env()
    yield e
    e.close()


def _guarded_query(e, pr, balls, k, sentinel, align=16, null_near=False, n=None):
    import test_memory_contract as M
    n = len(balls) if n is None else n
    outs = {"counts": n * 4}
    if not null_near:
        outs["near"] = max(n * k * 8, 0)
    got = M.run_call(e, lambda p: e.ctx.query_spheres_into(p["balls"], n, pr, k, None if null_near else p["near"], p["counts"]),
                     outs, ins={"balls": (balls, align)}, sentinel=sentinel, what=f"query_spheres k={k}")
    near = got["near"].view(np.int32).reshape(n, k, 2) if not null_near else np.zeros((n, k, 2), np.int32)
    return near[..., 0].view(F32), near[..., 1], got["counts"].view(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_guarded_outputs(env, name):
    s, cam = scene_named(name)
    pr = prepare(env.ctx, s, cam)
    balls = query_balls(s, 500, seed=3)
    want = brute(s, balls, 64)
    for k in (1, 7, 64):
        runs = [_guarded_query(env, pr, balls, k, sent, align=4 if k == 7 else 16) for sent in (0x00, 0xFF)]
        for r in runs:
            assert_same(r, first_k(want, k), f"guarded {name} k={k}")
    got = _guarded_query(env, pr, balls, 0, 0xFF, null_near=True)
    assert np.array_equal(got[2], want[2]), "k = 0 with near NULL"
    pr.free()


@pytest.mark.gpu
def test_poisoned_scratch(env):
    """The complete-box scratch of a stale scene is not trusted: results are the same whatever the pool held"""
    import test_memory_contract as M
    s, cam = scene_named("rgbbox")
    pr = prepare(env.ctx, s, cam)
    balls = query_balls(s, 500, seed=4)
    want = brute(s, balls, 8)
    e = env
    e.driver = M.Driver(0)
    try:
        for pattern in M.PATTERNS:
            e.pattern = pattern
            assert_same(_guarded_query(e, pr, balls, 8, 0x00), want, f"pattern {pattern:#x}")
    finally:
        e.pattern = None
    pr.free()


@pytest.mark.gpu
def test_errors_write_nothing(env):
    import test_memory_contract as M
    s, cam = scene_named("rgbbox")
    pr = prepare(env.ctx, s, cam)
    balls = query_balls(s, 64, seed=5)
    n = len(balls)
    lib, h = env.ctx.lib, env.ctx.handle
    calls = {
        "k = -1": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], n, -1, p["near"], p["counts"]),
        "k = 65": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], n, 65, p["near"], p["counts"]),
        "n < 0": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], -1, 8, p["near"], p["counts"]),
        "n > 2^30": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], (1 << 30) + 1, 8, p["near"], p["counts"]),
        "NULL balls": lambda p: lib.ray_b200_query_spheres(h, pr.handle, None, n, 8, p["near"], p["counts"]),
        "NULL near": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], n, 8, None, p["counts"]),
        "no output": lambda p: lib.ray_b200_query_spheres(h, pr.handle, p["balls"], n, 0, p["near"], None),
        "NULL scene": lambda p: lib.ray_b200_query_spheres(h, None, p["balls"], n, 8, p["near"], p["counts"]),
        "NULL batch": lambda p: lib.ray_b200_scene_batch_query_spheres(h, None, p["balls"], n, 8, p["near"], p["counts"]),
    }
    for what, call in calls.items():
        rcs = []
        got = M.run_call(env, lambda p: rcs.append(call(p)), {"near": n * 8 * 8, "counts": n * 4}, ins={"balls": (balls, 16)},
                         sentinel=0xFF, what=what)
        assert rcs[0] != 0, what
        assert env.ctx.get_error(), what
        assert (got["near"] == 0xFF).all() and (got["counts"] == 0xFF).all(), f"{what}: an output was written"
        assert_same(gpu_query(env.ctx, pr, balls, 8), brute(s, balls, 8), f"after {what}")   # the context stays usable
    assert lib.ray_b200_query_spheres(h, pr.handle, None, 0, 8, None, None) == 0            # n == 0 does nothing
    pr.free()


@pytest.mark.gpu
def test_stream_order_and_scenes_freed_in_flight():
    """Balls written by a producer on the context's stream are read after it; a scene freed or updated right after a
    query was enqueued still gives that query the old scene's answer"""
    import torch
    s, cam = RB.host_scene("random", 1 << 16, 4)
    s2, _ = RB.host_scene("random", 1 << 16, 5)
    balls = query_balls(s, 2000, seed=6)
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
            cnt = torch.empty((len(balls),), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(50_000_000)            # the producer is still running when the query is enqueued
                dst.copy_(src)
            c.query_spheres_into(dst.data_ptr(), len(balls), pr, 8, near.data_ptr(), cnt.data_ptr())
            if action == "free":
                pr.free()
            else:
                pr.update_from_ptr(s2_dev.data_ptr(), len(s2))
            c.sync()
            got = (near[..., 0].cpu().numpy(), near[..., 1].view(torch.int32).cpu().numpy(), cnt.cpu().numpy())
            assert_same(got, want, f"producer on the stream, scene {action}d in flight")
            if action == "update":
                assert_same(gpu_query(c, pr, balls, 8), brute(s2, balls, 8), "after the update")
                pr.free()
