"""The traversal kernels at the limits the library accepts: the deepest trees, 2^26 spheres, 2^30-pixel frames, ray
batches past 2^27 rays, path depth limits up to 65535, and exact-t ties.

Every test checks its own premise first (the depth reached, the sorted leaf indices hit, the offsets crossed, a tree only
partly staged), so that it cannot pass vacuously.  Results are compared bit for bit with the CPU oracle where its cost
is reasonable; for the largest scene, frame and ray batch, the independent paths cross-check each other: K0 (mega) does
not pack leaf indices into 26 bits, and the host builder is a second builder.

Depth limit: the stacks are sized for a tree depth of 63 (kStackSize), and render / the ray queries reject a deeper
tree.  No scene this library accepts gets there: the 30 Morton key bits give at most about 31 levels, and the index
tie-break of equal keys adds about log2 n more, so 2^26 spheres stay near 57.  That error cannot be triggered and has
no test.  The deepest scene here, the comb of limit_scenes.comb_scene, reaches 48.

The big tests print their wall time and the peak device memory in use (from cudaMemGetInfo, so it counts the library's
own allocations); run them with -s to see it.  They skip when the device does not have the memory free.
"""
import time

import numpy as np
import pytest

import limit_scenes as LS
import ray_query_oracle as Q
from test_ray_queries import bits_differ, hits_differ, quantise

GiB = 1 << 30


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


class DeviceUse:
    """Wall time and peak device memory in use (sampled at `mark`), printed at the end of a big test."""

    def __init__(self, what, need_gib):
        torch = _torch()
        torch.cuda.empty_cache()      # what earlier tests left in torch's cache is not this test's
        free, total = torch.cuda.mem_get_info()
        if free < need_gib * GiB:
            pytest.skip(f"{what} needs {need_gib} GiB of free device memory; {free / GiB:.1f} GiB are free")
        self.what, self.base, self.peak, self.t0 = what, total - free, 0, time.time()

    def mark(self):
        free, total = _torch().cuda.mem_get_info()
        self.peak = max(self.peak, total - free - self.base)

    def report(self):
        self.mark()
        print(f"\n[{self.what}] wall {time.time() - self.t0:.1f} s, peak device memory {self.peak / GiB:.2f} GiB")


def hit_records(h):
    """The dict of Context.trace_hits as float32[n][8] host records."""
    return np.concatenate([h["t"].cpu().numpy()[:, None], h["sphere"].cpu().numpy().view(np.float32)[:, None],
                           h["p"].cpu().numpy(), h["normal"].cpu().numpy()], 1)


def assert_frames_equal(got, want, what):
    bad = int((np.asarray(got) != np.asarray(want)).sum())
    assert bad == 0, f"{what}: {bad} of {np.asarray(want).size} pixels differ"


# ==================================================================================================== 1. deepest trees

COMB_M = 1 << 18            # cluster leaves at depth 30 + 18 = 48
COMB_DEPTH = 48
COMB_H, COMB_W = 48, 64


@pytest.fixture(scope="module")
def comb(oracle):
    s, first = LS.comb_scene(COMB_M)
    pr = oracle.Scene.custom(s, LS.COMB_CAM).prepare(COMB_H, COMB_W)
    tree = pr.dump()
    inner_depth, leaf_depth = LS.leaf_depths(tree)
    return dict(s=s, first=first, pr=pr, tree=tree, inner_depth=inner_depth, leaf_depth=leaf_depth)


def test_comb_tree_reaches_depth_48(R, comb):
    s, tree, leaf_depth = comb["s"], comb["tree"], comb["leaf_depth"]
    assert int(leaf_depth.max()) == COMB_DEPTH
    # the cluster is sorted first, in caller order (stable sort), and every one of its leaves is at the bottom
    np.testing.assert_array_equal(tree["perm"][:COMB_M], np.arange(COMB_M) + comb["first"])
    assert (tree["morton"][:COMB_M] == 0).all()
    assert (leaf_depth[:COMB_M] == COMB_DEPTH).all()
    # comb keys: the pair of bit b has key 1 << b, sorted right after the cluster
    want_keys = np.repeat(np.uint32(1) << np.arange(LS.COMB_LEVELS, dtype=np.uint32), 2)
    np.testing.assert_array_equal(tree["morton"][COMB_M:COMB_M + 60], want_keys)
    assert tree["morton"][-1] == LS.morton_of_cell(1023, 1023, 1023)
    # the spine: node at depth d < 30 has two inner children (the next spine node and the pair of the next bit down)
    node = 0
    for d in range(LS.COMB_LEVELS):
        left, right = int(tree["left"][node]), int(tree["right"][node])
        assert left >= 0 and right >= 0, d
        node = left
    assert comb["inner_depth"][node] == LS.COMB_LEVELS
    # the host builder agrees on every array and on the depth
    host = R.host_lbvh(s)
    for k in ("morton", "perm", "left", "right", "parent"):
        np.testing.assert_array_equal(host[k], tree[k], err_msg=k)
    np.testing.assert_array_equal(host["boxes"].view(np.uint32), tree["boxes"].view(np.uint32))
    assert host["max_depth"] == COMB_DEPTH


def test_comb_rays_defer_a_sibling_at_40_levels(R, comb):
    """Query rays and camera rays through the cluster pass both children's boxes at >= 40 levels on the way to the
    deepest leaves, so a stack walk holds >= 40 deferred siblings there."""
    tree, s = comb["tree"], comb["s"]
    for ray in LS.comb_query_rays(24, seed=1):
        assert LS.deferred_siblings(tree, s, ray, 0) >= 40, ray
    rays = R.camera_rays(tree["cam"], COMB_H, COMB_W).reshape(-1, 6)
    nested = [LS.deferred_siblings(tree, s, r, 0) for r in rays]
    assert sum(n >= 40 for n in nested) >= 10, sorted(nested)[-20:]


def test_comb_oracle_known_answers(comb):
    pr = Q.prepare_custom(comb["s"], LS.COMB_CAM, COMB_H, COMB_W)
    out = pr.trace_hits(LS.comb_query_rays(0, seed=1))
    for rec in out:
        d = -rec[2:5]
        assert rec[0] == 2.0 and rec[1:2].view(np.int32)[0] == comb["first"], rec
        assert np.abs(d).sum() == 1.0 and list(rec[5:8]) == list(-d), rec


COMB_K3 = [dict(wq_k=1), dict(wq_k=2), dict(wq_ncap=256), dict(wq_packet=1), dict(wq_packet=8), dict(wq_packet=32),
           dict(wq_k=2, wq_packet=8), dict(stage_cap=1024), dict(stage_cap=1024, wq_packet=8), dict(wq_low=-1),
           dict(wq_low=-1, wq_ncap=256)]
COMB_K5 = [dict(lw_slots=32), dict(lw_slots=48), dict(lw_slots=64), dict(lw_slots=32, lw_warps=4)]


@pytest.mark.gpu
def test_comb_on_gpu(R, comb):
    s, tree, pr_o = comb["s"], comb["tree"], comb["pr"]
    h, w = COMB_H, COMB_W
    want, _, cnt = pr_o.render(h, w)
    # the device build equals the oracle's tree, and its depth is the one computed above
    with R.Context() as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, LS.COMB_CAM))
        got = pr.dump()
        for k in ("morton", "perm", "left", "right", "parent"):
            np.testing.assert_array_equal(got[k], tree[k], err_msg=k)
        np.testing.assert_array_equal(got["boxes"].view(np.uint32), tree["boxes"].view(np.uint32))
        assert pr.info()["max_depth"] == int(comb["leaf_depth"].max()) == COMB_DEPTH
        work = ctx.count_work(h, w, pr)
        assert (work["segments"], work["box_tests"], work["leaf_tests"]) == (cnt["segments"], cnt["box_tests"], cnt["leaf_tests"])
        assert cnt["leaf_tests"] > 10 * COMB_M        # the frame does walk the cluster, many times
    runs = [dict(kernel=k) for k in ("mega", "persistent", "wavefront", "warpqueue", "streamqueue", "lanewalk")]
    runs += [dict(kernel="warpqueue", **t) for t in COMB_K3] + [dict(kernel="lanewalk", **t) for t in COMB_K5]
    for kw in runs:
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, LS.COMB_CAM))
            assert_frames_equal(ctx.render_host(h, w, pr), want, kw)


@pytest.mark.gpu
def test_comb_ray_queries_on_gpu(R, comb):
    s, tree, leaf_depth = comb["s"], comb["tree"], comb["leaf_depth"]
    rays = LS.comb_query_rays(122, seed=2)
    o = Q.prepare_custom(s, LS.COMB_CAM, COMB_H, COMB_W)
    want = o.trace_hits(rays)
    # premise: the winning leaves are the cluster's, at depth >= 45
    inv = np.empty_like(tree["perm"])
    inv[tree["perm"]] = np.arange(inv.shape[0], dtype=inv.dtype)
    won = want[:, 1].view(np.int32)
    assert (won >= 0).all() and (leaf_depth[inv[won]] >= 45).all()
    intervals = {(t_min, t_max): o.trace_hits(rays, t_min, t_max) for t_min, t_max in ((1.0, 100.0), (2.5, 1e9))}
    paths = {depth: o.trace_paths(rays, max_depth=depth) for depth in (1, 3, 50)}
    for kw in (dict(), dict(wq_k=2), dict(wq_ncap=256), dict(stage_cap=1024)):
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(COMB_H, COMB_W, ctx.scene_from_arrays(s, LS.COMB_CAM))
            d = _dev(rays)
            assert hits_differ(hit_records(ctx.trace_hits(pr, d)), want) == 0, kw
            for (t_min, t_max), want_i in intervals.items():
                assert hits_differ(hit_records(ctx.trace_hits(pr, d, t_min=t_min, t_max=t_max)), want_i) == 0, (kw, t_min)
            for depth, (want_rgb, want_seg) in paths.items():
                rgb, seg = ctx.trace_paths(pr, d, max_depth=depth)
                assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0, (kw, depth)
                assert (seg.cpu().numpy() == want_seg).all(), (kw, depth)


# ==================================================================================================== 2. 2^26 spheres

# The oracle is not used at this size: its (mostly single-threaded) builder took 95 s and 14.7 GB of host memory for the
# 2^26-sphere scene on an 8-core x86 host, against 21 s for the host builder.  K0 and the host builder are the cross-checks.
N26 = 1 << 26


def test_top_of_index_scene_premise(R):
    """The constructor of the 2^26 scene, at a size the CPU builds quickly: its targets are the last 32 sorted leaves."""
    n = 1 << 16
    s, cam, targets = LS.top_of_index_scene(n)
    t = R.host_lbvh(s)
    for j in range(LS.TOP_TARGETS):
        assert t["perm"][n - 1 - j] == targets[j]
    assert len(set(targets.tolist())) == LS.TOP_TARGETS
    assert t["morton"][n - LS.TOP_TARGETS - 1] < t["morton"][n - LS.TOP_TARGETS]
    o = Q.prepare_custom(s, cam, 64, 64)
    cases = LS.top_target_cases()
    out = o.trace_hits(np.array([c[0] for c in cases], np.float32))
    for j, (_, t_, p, nrm) in enumerate(cases):
        assert out[j, 0] == np.float32(t_) and out[j, 1:2].view(np.int32)[0] == targets[j]
        assert list(out[j, 2:5]) == list(np.float32(p)) and list(out[j, 5:8]) == list(np.float32(nrm))


@pytest.mark.gpu
def test_2pow26_spheres(R):
    torch = _torch()
    use = DeviceUse("2^26 spheres", 24)
    s, cam, targets = LS.top_of_index_scene(N26)
    h, w = 96, 128
    with R.Context(kernel="streamqueue") as ctx:     # the library with every kernel; set_kernel picks each in turn
        sc = ctx.scene_from_arrays(s, cam)
        pr = ctx.prepare_scene(h, w, sc)
        use.mark()
        info = pr.info()
        assert info["n_leaves"] == N26 and info["smem_nodes"] < info["n_inner"]
        got = pr.dump()
        use.mark()
        # premise: the targets are the last 32 leaves, i.e. at or above 2^26 - 32 (the top of the 26-bit index field)
        for j in range(LS.TOP_TARGETS):
            assert got["perm"][N26 - 1 - j] == targets[j]
        # the device build against the host build (a second builder): keys, order and sampled boxes
        host = R.host_lbvh(s)
        np.testing.assert_array_equal(got["morton"], host["morton"])
        np.testing.assert_array_equal(got["perm"], host["perm"])
        rng = np.random.default_rng(26)
        sample = np.concatenate([np.arange(64), rng.integers(0, N26 - 1, 100000), np.arange(N26 - 1 - 64, N26 - 1)])
        for k in ("left", "right", "parent"):
            np.testing.assert_array_equal(got[k][sample], host[k][sample], err_msg=k)
        np.testing.assert_array_equal(got["boxes"][sample].view(np.uint32), host["boxes"][sample].view(np.uint32))
        assert info["max_depth"] == host["max_depth"]
        del host, got
        # known answers of the targets
        cases = LS.top_target_cases()
        rays = _dev(np.array([c[0] for c in cases], np.float32))
        hits = hit_records(ctx.trace_hits(pr, rays))
        for j, (_, t, p, nrm) in enumerate(cases):
            assert hits[j, 0] == np.float32(t) and hits[j, 1:2].view(np.int32)[0] == targets[j], (j, hits[j])
            assert list(hits[j, 2:5]) == list(np.float32(p)) and list(hits[j, 5:8]) == list(np.float32(nrm)), (j, hits[j])
        rgb, seg = ctx.trace_paths(pr, rays)
        assert (seg.cpu().numpy() >= 2).all()      # every target reflects the ray upwards into the sky
        # frames: K3, K4 and K5 pack (slot, leaf index) into one word; K0 keeps the index whole
        frames = {}
        for k in ("mega", "warpqueue", "streamqueue", "lanewalk"):
            ctx.set_kernel(k)
            f = torch.empty((h, w), dtype=torch.int32, device="cuda")
            ctx.render_into(f.data_ptr(), h, w, pr)
            ctx.sync()
            frames[k] = f
            use.mark()
        ref = frames.pop("mega")
        assert len(torch.unique(ref)) > 100
        for k, f in frames.items():
            assert torch.equal(f, ref), k
        # one sphere more is refused, and the context stays usable
        s2 = np.concatenate([s, s[:1]])
        sc2 = ctx.scene_from_arrays(s2, cam)
        del s2
        with pytest.raises(R.RayError, match="too many spheres"):
            ctx.prepare_scene(h, w, sc2)
        sc2.free()
        ctx.set_kernel("warpqueue")
        again = hit_records(ctx.trace_hits(pr, rays))
        assert hits_differ(again, hits) == 0
    use.report()


# ==================================================================================================== 3. largest frames


def test_camera_rays_rows_equal_the_full_frame(R):
    pr = Q.prepare("irreg", 37, 91)
    full = R.camera_rays(pr.camera(), 37, 91).reshape(37, 91, 6)
    rows = [0, 5, 36]
    assert bits_differ(LS.camera_rays_rows(pr.camera(), 37, 91, rows), full[rows]) == 0
    # and at the largest frame size, against the oracle's get_ray
    h, w = 65536, 16384
    big = Q.prepare("irreg", h, w)
    got = LS.camera_rays_rows(big.camera(), h, w, [0, 32767, 65535])
    for a, j in enumerate([0, 32767, 65535]):
        for i in (0, 1, 8191, 16383):
            assert bits_differ(got[a, i], big.camera_ray(h, w, j, i)) == 0, (j, i)


def _tile_view(frame, world, rank):
    """The tiles rank `rank` of `world` renders, cut from a full h x w device frame (distributed.extract_rank_tiles)."""
    h, w = frame.shape
    t = frame.view(h // 4, 4, w // 8, 8).permute(0, 2, 1, 3).reshape(-1, 32)
    return t[rank::world]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(32768, 32768), (65536, 16384)])
def test_largest_frames(R, h, w):
    torch = _torch()
    use = DeviceUse(f"irreg {h}x{w}", 18)
    assert ((h + 3) // 4) * ((w + 7) // 8) == 1 << 25
    o = Q.prepare("irreg", h, w)
    rng = np.random.default_rng(h)
    rows = sorted({0, 1, h // 2, h - 2, h - 1, *rng.integers(0, h, 4).tolist()})
    want_rgb, _ = o.trace_paths(LS.camera_rays_rows(o.camera(), h, w, rows).reshape(-1, 6))
    want_rows = quantise(want_rgb).reshape(len(rows), w)
    a = torch.empty((h, w), dtype=torch.int32, device="cuda")
    b = torch.empty((h, w), dtype=torch.int32, device="cuda")
    with R.Context(kernel="mega") as ctx:
        pr = ctx.prepare_scene(h, w, ctx.irreg())
        ctx.render_into(a.data_ptr(), h, w, pr)
        ctx.sync()
    use.mark()
    assert_frames_equal(a[rows].cpu().numpy(), want_rows, "K0 rows vs oracle")
    for kw, frames in ((dict(), 1), (dict(learn_order=2), 2), (dict(heavy_first=1), 1)):
        with R.Context(kernel="warpqueue", **kw) as ctx:
            pr = ctx.prepare_scene(h, w, ctx.irreg())
            for k in range(frames):     # learn_order: the second frame claims its tiles in the order the first recorded
                b.fill_(-1)
                torch.cuda.synchronize()    # the context's own stream is not ordered after torch's
                ctx.render_into(b.data_ptr(), h, w, pr)
                ctx.sync()
                use.mark()
                assert torch.equal(a, b), (kw, k)
    del b
    world = 3
    with R.Context(kernel="warpqueue") as ctx:
        pr = ctx.prepare_scene(h, w, ctx.irreg())
        padded = ctx.shard_tiles_padded(h, w, world)
        tiles = torch.empty((padded, 32), dtype=torch.int32, device="cuda")
        for rank in range(world):
            count = ctx.shard_tiles(h, w, rank, world)
            tiles.fill_(-1)
            torch.cuda.synchronize()
            ctx.set_shard(rank, world)
            ctx.render_shard_into(tiles.data_ptr(), h, w, pr)
            ctx.sync()
            use.mark()
            assert torch.equal(tiles[:count], _tile_view(a, world, rank)), rank
        ctx.set_shard(0, 1)
        # one tile row or column more, or a side above 65536, is refused; the context stays usable
        for bh, bw in ((h, w + 8), (h + 4, w), (65537, 8), (8, 65537)):
            with pytest.raises(R.RayError, match="bad image size"):
                ctx.render(bh, bw, pr)
        small = ctx.render_host(64, 64, pr)
    assert_frames_equal(small, Q.prepare("irreg", h, w).render(64, 64)[0], "small frame after the errors")
    use.report()


# ==================================================================================================== 4. large ray batches

N28 = 1 << 28
SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes


@pytest.mark.gpu
def test_2pow28_rays(R):
    torch = _torch()
    use = DeviceUse("2^28 rays", 20)
    # premise: byte offsets of the rays (24 B) and of the hits (32 B) pass 4 GiB
    assert N28 * 24 > 4 * GiB and N28 * 32 > 4 * GiB
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
        # oracle subsample: mostly above 2^27, plus the last rays and a few from the start
        rng = np.random.default_rng(28)
        idx = np.unique(np.concatenate([rng.integers(1 << 27, N28, 6000), np.arange(N28 - 64, N28), rng.integers(0, 1 << 27, 500)]))
        sub = rays[torch.from_numpy(idx).cuda()].cpu().numpy()
        o = Q.prepare("irreg", 500, 500)
        hits = torch.full((N28, 8), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_hits_into(rays.data_ptr(), N28, pr, hits.data_ptr())
        ctx.sync()
        use.mark()
        assert not bool((hits == SENTINEL).any())
        got = hits[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.float32)
        want = o.trace_hits(sub)
        assert hits_differ(got, want) == 0
        assert (want[:, 0] > 0).mean() > 0.05
        del hits
        rgb = torch.full((N28, 3), SENTINEL, dtype=torch.int32, device="cuda")
        seg = torch.full((N28,), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_paths_into(rays.data_ptr(), N28, pr, rgb.data_ptr(), seg.data_ptr())
        ctx.sync()
        use.mark()
        assert not bool((rgb == SENTINEL).any()) and not bool((seg == SENTINEL).any())
        want_rgb, want_seg = o.trace_paths(sub)
        it = torch.from_numpy(idx).cuda()
        assert bits_differ(rgb[it].cpu().numpy().view(np.float32), want_rgb) == 0
        assert (seg[it].cpu().numpy() == want_seg).all()
    use.report()


# ==================================================================================================== 5. path depth limit

DEPTH_LIMITS = (1, 50, 51, 1000, 65535)
# (radius, gap, log2 offset range) of the facing spheres whose off-axis rays escape after the wanted segment counts
# (an escape after ~65535 segments needs mirrors so flat that float32 rounding pins the ray to the axis: the largest
# counts these scenes reach are a few thousand, so the limit 65535 is checked with the axis ray alone)
ESCAPE_SETS = [((5.0, 10.0, -2.6, 30), (1, 2, 3)),
               ((20.0, 2.0, 0, 100), (49, 50, 51, 52)),
               ((65536.0, 1.0, -6, 10), (999, 1000, 1001))]


@pytest.fixture(scope="module")
def escapes():
    """[(spheres, offsets {segments: offset})] found with the oracle (premise of the depth-limit test)."""
    out = []
    for (radius, gap, lo, hi), wanted in ESCAPE_SETS:
        s = LS.facing_spheres(radius, gap)
        pr = Q.prepare_custom(s, LS.FACING_CAM, 8, 8)
        out.append((s, LS.rays_escaping_after(pr, wanted, lo, hi), wanted))
    return out


def test_escape_rays_premise(escapes):
    for s, found, wanted in escapes:
        assert sorted(found) == sorted(wanted), (s[0, 6], found)
        pr = Q.prepare_custom(s, LS.FACING_CAM, 8, 8)
        for k, off in found.items():
            assert LS.bounce_count(pr, off) == (k, True)
    # the axis ray never escapes: every hit point, normal and reflection is exact
    pr = Q.prepare_custom(escapes[0][0], LS.FACING_CAM, 8, 8)
    assert LS.bounce_count(pr, 0.0) == (65535, False)


@pytest.mark.gpu
def test_path_depth_limits(R, escapes):
    for s, found, _ in escapes:
        o = Q.prepare_custom(s, LS.FACING_CAM, 8, 8)
        rays = np.array([LS.axis_ray(0.0)] + [LS.axis_ray(found[k]) for k in sorted(found)], np.float32)
        with R.Context() as ctx:
            pr = ctx.prepare_scene(8, 8, ctx.scene_from_arrays(s, LS.FACING_CAM))
            d = _dev(rays)
            for limit in DEPTH_LIMITS:
                rgb, seg = ctx.trace_paths(pr, d, max_depth=limit)
                rgb, seg = rgb.cpu().numpy(), seg.cpu().numpy()
                want_rgb, want_seg = o.trace_paths(rays, max_depth=limit)
                assert bits_differ(rgb, want_rgb) == 0 and (seg == want_seg).all(), limit
                # the ray on the axis runs into the limit: exactly `limit` objs_hit calls and no light
                assert seg[0] == limit and (rgb[0] == 0).all() and not np.signbit(rgb[0]).any(), limit
                for r, k in enumerate(sorted(found), start=1):   # escapes after k segments unless the limit comes first
                    assert seg[r] == min(k, limit), (limit, k)
                    assert bool(rgb[r].any()) == (k <= limit), (limit, k)


# ==================================================================================================== 6. ties


@pytest.fixture(scope="module")
def ties():
    s, groups = LS.tie_groups()
    return s, groups, Q.prepare_custom(s, LS.TIE_CAM, 96, 128)


def test_tie_groups_premise(R, ties):
    s, groups, _ = ties
    t = R.host_lbvh(s)
    inv = np.empty_like(t["perm"])
    inv[t["perm"]] = np.arange(inv.shape[0], dtype=inv.dtype)
    for g in groups:
        pos = np.sort(inv[g])
        assert (np.diff(pos) == 1).all() and (t["morton"][pos] == t["morton"][pos[0]]).all()
        assert t["perm"][pos[0]] == g.min()            # the lowest caller index is the lowest Morton leaf
        assert len(np.unique(s[g, 3:6], axis=0)) == len(g)   # every copy has its own colour
    assert not all((np.diff(g) == 1).all() for g in groups)   # the copies are scattered through the array


@pytest.mark.gpu
def test_tied_hits_report_the_lowest_index(R, ties):
    s, groups, o = ties
    rays = LS.tie_rays(len(groups))
    f = np.float32
    sky = lambda y: (f(1) - f(0.5) * (y + f(1))) * f(1) + f(0.5) * (y + f(1)) * np.float32([0.5, 0.7, 1.0])
    for kw in (dict(), dict(wq_k=2), dict(stage_cap=1024)):
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(96, 128, ctx.scene_from_arrays(s, LS.TIE_CAM))
            d = _dev(rays)
            got = hit_records(ctx.trace_hits(pr, d))
            assert hits_differ(got, o.trace_hits(rays)) == 0, kw
            for g, members in enumerate(groups):
                for a in range(4):
                    rec, ray = got[5 * g + a], rays[5 * g + a]
                    assert rec[0] == 4.0 and rec[1:2].view(np.int32)[0] == members.min(), (g, a, rec)
                    assert list(rec[2:5]) == list(ray[:3] + 20 * ray[3:] - 16 * ray[3:]), (g, a, rec)
                    assert list(rec[5:8]) == list(-ray[3:]), (g, a, rec)
            for t_min, t_max in ((0.0, 3.5), (3.5, 4.5), (3.9, 1e9), (4.0, 1e9), (5.0, 30.0), (0.05, 0.1)):
                got_i = hit_records(ctx.trace_hits(pr, d, t_min=t_min, t_max=t_max))
                assert hits_differ(got_i, o.trace_hits(rays, t_min, t_max)) == 0, (kw, t_min, t_max)
                if t_min < 4.0 < t_max:
                    assert (got_i[0::5, 1].view(np.int32) == [m.min() for m in groups]).all()
            rgb, seg = ctx.trace_paths(pr, d)
            rgb = rgb.cpu().numpy()
            want_rgb, want_seg = o.trace_paths(rays)
            assert bits_differ(rgb, want_rgb) == 0 and (seg.cpu().numpy() == want_seg).all(), kw
            for g, members in enumerate(groups):   # +z and -z rays reflect straight back into the horizon's sky
                for a in range(2):
                    assert list(rgb[5 * g + a]) == list(s[members.min(), 3:6] * sky(f(0))), (g, a)


TIE_FRAME = dict(h=72, w=96)
TIE_RUNS = ([dict(kernel="warpqueue", wq_packet=p, wq_k=k) for p in (1, 8, 16, 24, 32) for k in (1, 2)] +
            [dict(kernel="warpqueue"), dict(kernel="warpqueue", wq_k=2), dict(kernel="lanewalk"),
             dict(kernel="lanewalk", lw_slots=32), dict(kernel="mega")])


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 2])
def test_tied_frames(R, oracle, spp):
    """Tie groups of 2 to 100 copies in pixel frames, with the packet walk on explicitly and through `auto`.  The filler
    makes the tree larger than the staging area, so `auto` (spp > 1: coherent rays) turns the packet walk on."""
    s, groups = LS.tie_groups(filler=30000)
    h, w = TIE_FRAME["h"], TIE_FRAME["w"]
    o = oracle.Scene.custom(s, LS.TIE_CAM).prepare(h, w)
    want, _, _ = o.render(h, w, spp=spp)
    # premise: many primary rays win on a tie group (whose copies have different colours), each group is seen
    cam = o.dump()["cam"]
    first = Q.prepare_custom(s, LS.TIE_CAM, h, w).trace_hits(R.camera_rays(cam, h, w).reshape(-1, 6))[:, 1].view(np.int32)
    for g in groups:
        assert np.isin(first, g).sum() >= 20, len(g)
    for kw in TIE_RUNS:
        with R.Context(**kw) as ctx:
            pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, LS.TIE_CAM))
            info = pr.info()
            assert info["smem_nodes"] < info["n_inner"], kw
            assert_frames_equal(ctx.render_host(h, w, pr, spp=spp), want, kw)
