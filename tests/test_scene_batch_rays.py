"""Ray queries of scene batches (include/ray_b200.h "scene batches"): m rays per scene of a batch of B scenes, traced in
one launch to their closest hits, along their paths, to occlusion or to their k nearest hits, per call or with per-ray
intervals.  The answer for ray j of scene b is bit for bit the single-scene query's for that ray on member b, and on an
independently prepared scene of the same records; sphere indexes scene b's own records.

On the CPU: the Python argument checks, the query names and the binding.  On the GPU: every kind on mixed batches
against members, independent scenes and the CPU oracle; batch sizes, scene isolation, the carried-over identities, every
instantiation of the three kinds, 64-bit record offsets, stream order, freeing, guarded outputs, poisoned pools and
errors."""
import os
import re

import numpy as np
import pytest

import ray_query_oracle as Q
from ray_query_cases import INTERVALS, T24, _dev, _np, _torch, bits_differ, hits_differ, max_hit_t, random_rays
from test_scene_batch import STAGING, mixed_batch, random_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 24, 32
SENT = 0x7FA5A5A5
BATCH_SYMBOLS = [f"ray_b200_scene_batch_trace_{q}" for q in ("hits", "paths", "occluded", "multi_hits", "hits_ranged",
                                                             "occluded_ranged", "multi_hits_ranged")]
PLAN_QUERY = {"hits": "scene_batch_closest", "paths": "scene_batch_closest", "occluded": "scene_batch_anyhit",
              "multi_hits": "scene_batch_multihit"}
# per-ray intervals of the ranged rays: valid ones, empty ones and ones the per-call forms reject
RAY_INTERVALS = INTERVALS + [(0.0, 0.0), (5.0, 2.0), (0.1, 3.0), (-1.0, 1e9), (np.nan, 1e9), (np.inf, 1e9), (0.0, np.nan),
                             (0.0, np.inf), (0.0, -np.inf), (-0.0, 1e9)]


# ------------------------------------------------------------------------------------------ rays


def scene_rays(spheres, m, seed):
    """m rays of one scene: half random (random_rays over its finite records), half aimed from there at a sphere's centre"""
    s = np.asarray(spheres, np.float32)
    ok = np.isfinite(s).all(1) & (np.abs(s[:, [0, 1, 2, 6]]).max(1) < 1e6)
    src = s[ok] if ok.any() else np.float32([[0, 0, 0, 0, 0, 0, 1]])
    r = random_rays(src, m, seed)
    rng = np.random.default_rng(seed + 1)
    aim = rng.random(m) < 0.5
    c = src[rng.integers(0, len(src), m), :3]
    r[aim, 3:6] = c[aim] - r[aim, :3]
    return r


def batch_rays(spheres, m, seed):
    """[B, m, 6] rays, scene b's from scene_rays of its records"""
    return np.ascontiguousarray(np.stack([scene_rays(sb, m, seed + 7 * b) for b, sb in enumerate(spheres)]), np.float32)


def ranged(rays6, seed):
    """[..., 8] rays (origin, t_min, direction, t_max) with intervals drawn from RAY_INTERVALS"""
    r = np.asarray(rays6, np.float32)
    iv = np.array(RAY_INTERVALS, np.float32)[np.random.default_rng(seed).integers(0, len(RAY_INTERVALS), r.shape[:-1])]
    return np.ascontiguousarray(np.concatenate([r[..., :3], iv[..., :1], r[..., 3:], iv[..., 1:]], -1), np.float32)


# ------------------------------------------------------------------------------------------ queries as host arrays


def _out(shape, dtype="f"):
    torch = _torch()
    if dtype == "u8":
        return torch.full(shape, 0xA5, dtype=torch.uint8, device="cuda")
    t = torch.full(shape, SENT, dtype=torch.int32, device="cuda")
    return t.view(torch.float32) if dtype == "f" else t


def _host(out):
    return {k: _np(v) for k, v in out.items()}


def run_batch(ctx, batch, kind, rays, k=4, t=(0.0, 1e9), max_depth=50):
    """A batch query through the raw form on sentinel-filled outputs: {records / rgb, segments / occluded / counts} as
    host arrays of shape [B, m, ...]"""
    torch = _torch()
    B, m, width = rays.shape
    rg, p = width == 8, rays.data_ptr()
    torch.cuda.synchronize()
    if kind == "hits":
        o = {"records": _out((B, m, 8))}
        if rg:
            ctx.trace_scene_batch_hits_ranged_into(p, m, batch, o["records"].data_ptr())
        else:
            ctx.trace_scene_batch_hits_into(p, m, batch, o["records"].data_ptr(), *t)
    elif kind == "paths":
        o = {"rgb": _out((B, m, 3)), "segments": _out((B, m), "i")}
        ctx.trace_scene_batch_paths_into(p, m, batch, o["rgb"].data_ptr(), o["segments"].data_ptr(), max_depth=max_depth)
    elif kind == "occluded":
        o = {"occluded": _out((B, m), "u8")}
        if rg:
            ctx.trace_scene_batch_occluded_ranged_into(p, m, batch, o["occluded"].data_ptr())
        else:
            ctx.trace_scene_batch_occluded_into(p, m, batch, o["occluded"].data_ptr(), *t)
    else:
        o = {"records": _out((B, m, k, 8)), "counts": _out((B, m), "i")}
        if rg:
            ctx.trace_scene_batch_multi_hits_ranged_into(p, m, batch, k, o["records"].data_ptr(), o["counts"].data_ptr())
        else:
            ctx.trace_scene_batch_multi_hits_into(p, m, batch, k, o["records"].data_ptr(), o["counts"].data_ptr(), *t)
    ctx.sync()
    return _host(o)


def run_single(ctx, pr, kind, rays, k=4, t=(0.0, 1e9), max_depth=50):
    """The single-scene query of [m, 6 | 8] rays on a prepared scene, in run_batch's form with shape [m, ...]"""
    torch = _torch()
    m, width = rays.shape
    rg, p = width == 8, rays.data_ptr()
    torch.cuda.synchronize()
    if kind == "hits":
        o = {"records": _out((m, 8))}
        if rg:
            ctx.trace_hits_ranged_into(p, m, pr, o["records"].data_ptr())
        else:
            ctx.trace_hits_into(p, m, pr, o["records"].data_ptr(), *t)
    elif kind == "paths":
        o = {"rgb": _out((m, 3)), "segments": _out((m,), "i")}
        ctx.trace_paths_into(p, m, pr, o["rgb"].data_ptr(), o["segments"].data_ptr(), max_depth=max_depth)
    elif kind == "occluded":
        o = {"occluded": _out((m,), "u8")}
        if rg:
            ctx.trace_occluded_ranged_into(p, m, pr, o["occluded"].data_ptr())
        else:
            ctx.trace_occluded_into(p, m, pr, o["occluded"].data_ptr(), *t)
    else:
        o = {"records": _out((m, k, 8)), "counts": _out((m,), "i")}
        if rg:
            ctx.trace_multi_hits_ranged_into(p, m, pr, k, o["records"].data_ptr(), o["counts"].data_ptr())
        else:
            ctx.trace_multi_hits_into(p, m, pr, k, o["records"].data_ptr(), o["counts"].data_ptr(), *t)
    ctx.sync()
    return _host(o)


def run_oracle(o, kind, rays, k=4, t=(0.0, 1e9), max_depth=50):
    """The CPU oracle's answer in run_batch's form (host rays [m, 6 | 8])"""
    rg = rays.shape[1] == 8
    if kind == "hits":
        return {"records": o.trace_hits_ranged(rays) if rg else o.trace_hits(rays, *t)}
    if kind == "paths":
        rgb, seg = o.trace_paths(rays, max_depth)
        return {"rgb": rgb, "segments": seg}
    if kind == "occluded":
        return {"occluded": (o.trace_occluded_ranged(rays) if rg else o.trace_occluded(rays, *t)).view(np.uint8)}
    rec, cnt = o.trace_multi_hits_ranged(rays, k) if rg else o.trace_multi_hits(rays, k, *t)
    return {"records": rec, "counts": cnt}


def assert_same(got, want, what):
    for key, w in want.items():
        g = got[key]
        if key == "records":
            bad = hits_differ(g.reshape(-1, 8), w.reshape(-1, 8))
        elif key == "rgb":
            bad = bits_differ(g, w)
        else:
            bad = int((np.asarray(g).reshape(-1) != np.asarray(w).reshape(-1)).sum())
        assert bad == 0, f"{what}: {bad} {key} values differ"


def assert_local_spheres(got, n, what):
    if "records" in got:
        sph = np.ascontiguousarray(got["records"][..., 1]).view(np.int32)
        assert ((sph == -1) | ((sph >= 0) & (sph < n))).all(), f"{what}: sphere outside [0, {n}) or -1"


def cases(rays6, rays8, k, t, max_depth):
    """(kind, rays, keyword arguments) of every entry point"""
    return [("hits", rays6, dict(t=t)), ("paths", rays6, dict(max_depth=max_depth)), ("occluded", rays6, dict(t=t)),
            ("multi_hits", rays6, dict(k=k, t=t)), ("hits", rays8, {}), ("occluded", rays8, {}), ("multi_hits", rays8, dict(k=k))]


# ------------------------------------------------------------------------------------------ CPU


class FakeBatch:
    shape = (3, 5)


def test_python_argument_checks(R):
    torch = _torch()

    class NoContext:   # the argument checks only, without a device
        device = 0
        _batch_rays_tensor = R.Context._batch_rays_tensor
    r6 = np.zeros((3, 4, 6), np.float32)
    C = R.Context
    tensor_forms = (C.trace_scene_batch_hits, C.trace_scene_batch_occluded, C.trace_scene_batch_paths)
    bad = [r6, None, torch.from_numpy(r6), torch.from_numpy(r6[0]), torch.from_numpy(r6[..., :5].copy()),
           torch.from_numpy(np.zeros((3, 4, 7), np.float32)), torch.from_numpy(r6.astype(np.float64)),
           torch.empty((3, 4, 6), device="meta"), torch.from_numpy(np.zeros((3, 4, 6, 1), np.float32))]
    for f in tensor_forms:
        for rays in bad:
            with pytest.raises(ValueError):
                f(NoContext(), FakeBatch(), rays)
    for rays in bad:
        with pytest.raises(ValueError):
            C.trace_scene_batch_multi_hits(NoContext(), FakeBatch(), rays, 4)
    r8 = torch.from_numpy(np.zeros((3, 4, 8), np.float32))
    with pytest.raises(ValueError, match="own"):
        C.trace_scene_batch_hits(NoContext(), FakeBatch(), r8, t_min=0.1)
    with pytest.raises(ValueError, match="own"):
        C.trace_scene_batch_multi_hits(NoContext(), FakeBatch(), r8, 2, t_max=5.0)
    with pytest.raises(ValueError, match=r"\[B, m, 6\]"):
        C.trace_scene_batch_paths(NoContext(), FakeBatch(), r8)   # paths have no ranged form
    if not torch.cuda.is_available():
        return
    d6 = torch.zeros((3, 4, 6), device="cuda")
    for rays in (d6.double(), d6.transpose(0, 1).contiguous().transpose(0, 1), d6[:, ::2], d6[:2], torch.zeros((4, 4, 6), device="cuda"),
                 torch.zeros((3, 4, 8), device="cuda").half()):
        for f in tensor_forms:
            with pytest.raises(ValueError):
                f(NoContext(), FakeBatch(), rays)
    with pytest.raises(ValueError, match="own"):
        C.trace_scene_batch_occluded(NoContext(), FakeBatch(), torch.zeros((3, 4, 8), device="cuda"), t_min=0.0)
    with pytest.raises(ValueError, match="one row per scene"):
        C.trace_scene_batch_hits(NoContext(), FakeBatch(), torch.zeros((2, 4, 6), device="cuda"))


def test_query_names_match_the_header(R):
    assert R.QUERIES[10:13] == ("scene_batch_closest", "scene_batch_anyhit", "scene_batch_multihit")
    text = open(os.path.join(ROOT, "include", "ray_b200.h")).read()
    enum = re.search(r"enum ray_b200_query \{(.*?)\}", text, flags=re.S).group(1)
    values = dict(re.findall(r"RAY_B200_QUERY_(\w+) = (\d+)", enum))
    assert {k: int(v) for k, v in values.items() if k.startswith("SCENE_BATCH_")} == {
        "SCENE_BATCH_CLOSEST": 10, "SCENE_BATCH_ANYHIT": 11, "SCENE_BATCH_MULTIHIT": 12}


def test_header_declares_and_binding_binds_the_batch_queries(R):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ray_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ray_b200_\w+)\s*\(", text))
    assert set(BATCH_SYMBOLS) <= declared
    assert set(BATCH_SYMBOLS) <= set(R.declared_symbols())
    import ctypes
    lib = ctypes.CDLL(R.lib_path())
    assert all(hasattr(lib, f) for f in BATCH_SYMBOLS)


# ------------------------------------------------------------------------------------------ GPU: exactness


def check_batch(ctx, batch, s, rays6, rays8, k, t, max_depth, refs, oracles=None, members=None, what=""):
    """Every entry point on the batch against run_single on each scene's prepared scenes in refs, and against the oracle
    where oracles is given"""
    B, m = rays6.shape[:2]
    n = s.shape[1]
    d6, d8 = _dev(rays6), _dev(rays8)
    for kind, rays, kw in cases(d6, d8, k, t, max_depth):
        rg = rays.shape[2] == 8
        n0 = ctx.launch_count()
        got = run_batch(ctx, batch, kind, rays, **kw)
        tag = f"{what} {kind}{' ranged' if rg else ''} m={m} {kw}"
        if m > 0 and not (kind == "paths" and max_depth == 0):
            plan = ctx.last_plan()
            assert ctx.launch_count() - n0 == 1, tag
            assert plan["query"] == PLAN_QUERY[kind] and plan["ranged"] == int(rg), (tag, plan)
            assert plan["n_inner"] == B * (n - 1) and plan["n_leaves"] == B * n, (tag, plan)
        else:
            assert ctx.launch_count() == n0, tag
        assert_local_spheres(got, n, tag)
        for b in (members if members is not None else range(B)):
            mine = {key: v[b] for key, v in got.items()}
            for ref_name, prs in refs.items():
                want = run_single(ctx, prs[b], kind, rays[b], **kw)
                assert_same(mine, want, f"{tag} scene {b} vs {ref_name}")
            if oracles is not None:
                want = run_oracle(oracles[b], kind, (rays8 if rg else rays6)[b], **kw)
                assert_same(mine, want, f"{tag} scene {b} vs the oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 64, 1000])
def test_mixed_batch_every_kind_equals_members_and_independent_scenes(R, n):
    s, cams = mixed_batch(n)
    B = len(s)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        refs = {"member": [batch.member(b) for b in range(B)],
                "independent": [ctx.prepare_scene_device(H, W, _dev(s[b]), cams[b]) for b in range(B)]}
        for i, (m, k, depth) in enumerate(((1, 1, 0), (3, 7, 1), (31, 64, 3), (1000, 7, 50), (0, 4, 50))):
            r6 = batch_rays(s, m, seed=100 * n + i)
            r8 = ranged(r6, seed=i)
            oracles = [Q.prepare_custom(s[b], cams[b], H, W) for b in range(B)] if n <= 64 and 0 < m <= 31 else None
            check_batch(ctx, batch, s, r6, r8, k, INTERVALS[i % len(INTERVALS)], depth, refs, oracles, what=f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,m", [(1, 64, 1000), (2, 3, 31), (7, 1000, 3), (1024, 64, 31), (1024, 2, 1)])
def test_batch_sizes(R, B, n, m):
    s, cams = random_batch(B, n, seed=B + n + m)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        sample = range(B) if B <= 8 else sorted({0, 1, B // 3, B // 2, B - 2, B - 1})
        refs = {"member": {b: batch.member(b) for b in sample},
                "independent": {b: ctx.prepare_scene_device(H, W, _dev(s[b]), cams[b]) for b in sample}}
        r6 = batch_rays(s, m, seed=B)
        for t, k, depth in (((0.0, 1e9), 7, 50), ((0.1, 40.0), 64, 3), ((2.5, 1e9), 1, 1)):
            check_batch(ctx, batch, s, r6, ranged(r6, seed=k), k, t, depth, refs, members=sample, what=f"B={B} n={n}")


@pytest.mark.gpu
def test_scene_isolation(R):
    """Every member fills the same cube with different spheres and every scene's rays are the same: a ray that reached
    another scene's tree, or a sphere index not made local, gives a plausible answer that is not the member's."""
    B, n, m = 9, 200, 500
    rng = np.random.default_rng(4)
    s = np.empty((B, n, 7), np.float32)
    s[:, :, 0:3] = rng.uniform(-10, 10, (B, n, 3))
    s[:, :, 3:6] = rng.uniform(0.2, 0.9, (B, n, 3))
    s[:, :, 6] = rng.uniform(0.3, 1.5, (B, n))
    cams = np.tile(np.float32([0, 0, 40, 0, 0, 0, 50]), (B, 1))
    r = scene_rays(s.reshape(-1, 7), m, seed=3)
    r6 = np.ascontiguousarray(np.broadcast_to(r, (B, m, 6)), np.float32)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        refs = {"member": [batch.member(b) for b in range(B)]}
        oracles = [Q.prepare_custom(s[b], cams[b], H, W) for b in range(B)]
        check_batch(ctx, batch, s, r6, ranged(r6, seed=2), 8, (0.0, 1e9), 50, refs, oracles, what="isolation")
        got = run_batch(ctx, batch, "hits", _dev(r6))
        sph = np.ascontiguousarray(got["records"][..., 1]).view(np.int32)
        assert (sph >= 0).mean() > 0.3
        assert (sph[1:] != sph[:1]).any(1).all(), "every scene answers differently from scene 0"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 1000])
def test_identities_carry_over(R, n):
    """counts > 0 == occluded on mixed batches, and record 0 of multi-hit at t_min = 0.1 is trace_hits' record on scenes
    whose hits all have t < 2^24"""
    s, cams = mixed_batch(n)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        r6 = batch_rays(s, 700, seed=n)
        d6 = _dev(r6)
        for t in INTERVALS:
            occ = run_batch(ctx, batch, "occluded", d6, t=t)["occluded"]
            mh = run_batch(ctx, batch, "multi_hits", d6, k=3, t=t)
            assert ((mh["counts"] > 0) == (occ == 1)).all(), t
        d8 = _dev(ranged(r6, seed=5))
        occ = run_batch(ctx, batch, "occluded", d8)["occluded"]
        assert ((run_batch(ctx, batch, "multi_hits", d8, k=2)["counts"] > 0) == (occ == 1)).all()
    s, cams = random_batch(6, n, seed=n)
    r6 = batch_rays(s, 700, seed=n + 1)
    assert max(max_hit_t(s[b], r6[b]) for b in range(len(s))) < T24   # premise: the re-intersection of trace_hits cannot fail
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        d6 = _dev(r6)
        for t_max in (1e9, 20.0):
            hits = run_batch(ctx, batch, "hits", d6, t=(0.1, t_max))["records"]
            first = run_batch(ctx, batch, "multi_hits", d6, k=1, t=(0.1, t_max))["records"][:, :, 0]
            assert (hits[..., 0] > 0).sum() > 100
            assert hits_differ(first.reshape(-1, 8), hits.reshape(-1, 8)) == 0, t_max


@pytest.mark.gpu
def test_every_plan_of_the_kinds(R):
    """Forced staging (partial, nodes, whole) x K = 1 / 2 x per-call / ranged x the three kinds: all 36 variants are
    launched, and every answer equals the single-scene query's on the members."""
    B, n, m = 8, 60, 300
    s, cams = random_batch(B, n, seed=11)
    n_inner, n_leaves = B * (n - 1), B * n
    caps = {"partial": 64 * (n_inner // 3), "nodes": 64 * n_inner + 128, "whole": 64 * n_inner + 16 * n_leaves + 256}
    r6 = batch_rays(s, m, seed=1)
    r8 = ranged(r6, seed=1)
    with R.Context() as ref:
        prs = [ref.prepare_scene_device(H, W, _dev(s[b]), cams[b]) for b in range(B)]
        d6, d8 = _dev(r6), _dev(r8)
        want = {}
        for kind, rays, kw in cases(d6, d8, 5, (0.1, 1e9), 50):
            want[kind, rays.shape[2] == 8] = [run_single(ref, prs[b], kind, rays[b], **kw) for b in range(B)]
    launched = set()
    for plan_kw in (dict(wq_k=1, wq_warps=32), dict(wq_k=2, wq_warps=16)):
        for stage, cap in caps.items():
            with R.Context(stage_cap=cap, wq_ncap=256, **plan_kw) as ctx:
                batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
                d6, d8 = _dev(r6), _dev(r8)
                for kind, rays, kw in cases(d6, d8, 5, (0.1, 1e9), 50):
                    rg = rays.shape[2] == 8
                    got = run_batch(ctx, batch, kind, rays, **kw)
                    plan = ctx.last_plan()
                    what = f"{plan_kw} {stage} {kind} ranged={rg}"
                    assert plan["query"] == PLAN_QUERY[kind] and STAGING[(plan["all_nodes"], plan["spheres"])] == stage, (what, plan)
                    assert plan["k"] == plan_kw["wq_k"] and plan["ranged"] == int(rg), (what, plan)
                    launched.add((plan["k"], stage, rg, plan["query"]))
                    for b in range(B):
                        assert_same({key: v[b] for key, v in got.items()}, want[kind, rg][b], f"{what} scene {b}")
    reachable = {(k, st, rg, q) for k in (1, 2) for st in STAGING.values() for rg in (False, True)
                 for q in ("scene_batch_closest", "scene_batch_anyhit", "scene_batch_multihit")}
    assert launched == reachable, reachable - launched


@pytest.mark.gpu
def test_multi_hit_records_past_4_gib(R):
    """B m k records of 32 bytes pass 4 GiB: the last scene's records land at their 64-bit offsets."""
    torch = _torch()
    B, n, k = 2, 300, 64
    m = (1 << 20) + 4096            # 2 x (2^20 + 4096) x 64 x 32 bytes = 4.03 GiB
    s, cams = random_batch(B, n, seed=6)
    tail = 2048
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        r6 = np.ascontiguousarray(np.stack([np.tile(scene_rays(s[b], tail, seed=b), (m // tail + 1, 1))[:m] for b in range(B)]),
                                  np.float32)
        d6 = _dev(r6)
        rec = torch.empty((B, m, k, 8), dtype=torch.float32, device="cuda")
        cnt = torch.empty((B, m), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_scene_batch_multi_hits_into(d6.data_ptr(), m, batch, k, rec.data_ptr(), cnt.data_ptr())
        ctx.sync()
        for b in range(B):
            pr = batch.member(b)
            want = run_single(ctx, pr, "multi_hits", d6[b, m - tail:].contiguous(), k=k)
            got = {"records": _np(rec[b, m - tail:]), "counts": _np(cnt[b, m - tail:])}
            assert_same(got, want, f"scene {b}, the last {tail} rays")
            assert (want["counts"] > 0).any()
        del rec, cnt


# ------------------------------------------------------------------------------------------ GPU: order and memory


@pytest.mark.gpu
def test_queries_in_flight_read_the_old_trees_and_free_behind_them(R):
    torch = _torch()
    B, n, m = 8, 2000, 1 << 16
    s, cams = random_batch(B, n, seed=4)
    s2 = s.copy()
    s2[:, :, 0:3] += 3.0
    r6 = batch_rays(s, m, seed=9)
    with R.Context() as ctx:
        d6 = _dev(r6)
        old = run_batch(ctx, ctx.prepare_scene_batch(H, W, _dev(s), cams), "multi_hits", d6, k=4)
        new = run_batch(ctx, ctx.prepare_scene_batch(H, W, _dev(s2), cams), "multi_hits", d6, k=4)
        assert (old["counts"] != new["counts"]).any()
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        outs = [(torch.empty((B, m, 4, 8), device="cuda"), torch.empty((B, m), dtype=torch.int32, device="cuda")) for _ in range(2)]
        torch.cuda.synchronize()
        ctx.trace_scene_batch_multi_hits_into(d6.data_ptr(), m, batch, 4, outs[0][0].data_ptr(), outs[0][1].data_ptr())
        batch.update(_dev(s2))
        ctx.trace_scene_batch_multi_hits_into(d6.data_ptr(), m, batch, 4, outs[1][0].data_ptr(), outs[1][1].data_ptr())
        batch.free()                      # with the second query possibly still running
        ctx.sync()
        for (rec, cnt), want in zip(outs, (old, new)):
            assert_same({"records": _np(rec), "counts": _np(cnt)}, want, "in flight")


@pytest.mark.gpu
def test_guarded_outputs_and_untouched_rays(R):
    from test_memory_contract import Guarded
    B, n, m, k = 3, 40, 37, 7
    s, cams = random_batch(B, n, seed=5)
    r6 = batch_rays(s, m, seed=5)
    r8 = ranged(r6, seed=5)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        for kind, rays, kw in cases(r6, r8, k, (0.1, 1e9), 3):
            rg = rays.shape[2] == 8
            want = run_batch(ctx, batch, kind, _dev(rays), **kw)
            for fill in (0x00, 0xFF):
                rin = Guarded(0, fill, align=4 if rg else 16, data=rays)
                if kind in ("hits", "multi_hits"):
                    outs = {"records": Guarded(B * m * (k if kind == "multi_hits" else 1) * 32, fill)}
                    if kind == "multi_hits":
                        outs["counts"] = Guarded(B * m * 4, fill)
                elif kind == "paths":
                    outs = {"rgb": Guarded(B * m * 12, fill), "segments": Guarded(B * m * 4, fill)}
                else:
                    outs = {"occluded": Guarded(B * m, fill)}
                p = {key: g.ptr for key, g in outs.items()}
                _torch().cuda.synchronize()
                if kind == "hits":
                    (ctx.trace_scene_batch_hits_ranged_into(rin.ptr, m, batch, p["records"]) if rg else
                     ctx.trace_scene_batch_hits_into(rin.ptr, m, batch, p["records"], *kw["t"]))
                elif kind == "paths":
                    ctx.trace_scene_batch_paths_into(rin.ptr, m, batch, p["rgb"], p["segments"], max_depth=kw["max_depth"])
                elif kind == "occluded":
                    (ctx.trace_scene_batch_occluded_ranged_into(rin.ptr, m, batch, p["occluded"]) if rg else
                     ctx.trace_scene_batch_occluded_into(rin.ptr, m, batch, p["occluded"], *kw["t"]))
                else:
                    (ctx.trace_scene_batch_multi_hits_ranged_into(rin.ptr, m, batch, k, p["records"], p["counts"]) if rg else
                     ctx.trace_scene_batch_multi_hits_into(rin.ptr, m, batch, k, p["records"], p["counts"], *kw["t"]))
                ctx.sync()
                what = f"{kind} ranged={rg} fill {fill:#x}"
                assert np.array_equal(rin.check(f"{what} rays"), np.ascontiguousarray(rays).view(np.uint8).reshape(-1)), what
                got = {}
                for key, g in outs.items():
                    body = g.check(f"{what} {key}")
                    got[key] = body if key == "occluded" else body.view(np.int32 if key in ("counts", "segments") else np.float32)
                assert_same(got, {key: v.reshape(-1) if key != "records" else v for key, v in want.items()}, what)


@pytest.mark.gpu
@pytest.mark.parametrize("poison", [0x00, 0xFF, 0x7F])
def test_outputs_do_not_depend_on_pool_contents(R, poison):
    from test_memory_contract import Driver
    torch = _torch()
    B, n, m = 5, 300, 500
    s, cams = random_batch(B, n, seed=13)
    r6 = batch_rays(s, m, seed=13)
    r8 = ranged(r6, seed=13)
    with R.Context() as ref:
        batch = ref.prepare_scene_batch(H, W, _dev(s), cams)
        want = [run_batch(ref, batch, kind, rays, **kw) for kind, rays, kw in cases(_dev(r6), _dev(r8), 6, (0.0, 1e9), 50)]
    drv = Driver(0)
    st = torch.cuda.Stream()
    with R.Context() as ctx, torch.cuda.stream(st):
        ctx.set_stream(st.cuda_stream)
        d6, d8 = _dev(r6), _dev(r8)
        st.synchronize()
        drv.poison_pool(st.cuda_stream, poison)
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        for (kind, rays, kw), w in zip(cases(d6, d8, 6, (0.0, 1e9), 50), want):
            drv.poison_pool(st.cuda_stream, poison)
            assert_same(run_batch(ctx, batch, kind, rays, **kw), w, f"{kind} poison {poison:#x}")
        batch.free()
        ctx.set_stream(None)


# ------------------------------------------------------------------------------------------ GPU: errors


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    B, n, m = 3, 20, 16
    s, cams = random_batch(B, n, seed=2)
    r6 = batch_rays(s, m, seed=2)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        d6, d8 = _dev(r6), _dev(ranged(r6, seed=2))
        want = {kind: run_batch(ctx, batch, kind, rays, **kw) for kind, rays, kw in cases(d6, d8, 4, (0.0, 1e9), 50)[:4]}
        out = torch.empty((B, m, 64, 8), device="cuda")
        p, o = d6.data_ptr(), out.data_ptr()

        class Freed:
            handle = None

        calls = [lambda: ctx.trace_scene_batch_hits_into(p, m, batch, o, -1.0, 1e9),
                 lambda: ctx.trace_scene_batch_hits_into(p, m, batch, o, np.nan, 1e9),
                 lambda: ctx.trace_scene_batch_occluded_into(p, m, batch, o, 0.0, np.inf),
                 lambda: ctx.trace_scene_batch_multi_hits_into(p, m, batch, 0, o),
                 lambda: ctx.trace_scene_batch_multi_hits_into(p, m, batch, 65, o),
                 lambda: ctx.trace_scene_batch_multi_hits_ranged_into(d8.data_ptr(), m, batch, 0, o),
                 lambda: ctx.trace_scene_batch_paths_into(p, m, batch, o, max_depth=-1),
                 lambda: ctx.trace_scene_batch_paths_into(p, m, batch, o, max_depth=65536),
                 lambda: ctx.trace_scene_batch_hits_into(None, m, batch, o),
                 lambda: ctx.trace_scene_batch_hits_into(p, m, batch, None),
                 lambda: ctx.trace_scene_batch_occluded_ranged_into(d8.data_ptr(), m, batch, None),
                 lambda: ctx.trace_scene_batch_hits_into(p, m, Freed(), o),                      # NULL batch
                 lambda: ctx.trace_scene_batch_hits_into(p, -1, batch, o),                       # m < 0
                 lambda: ctx.trace_scene_batch_hits_into(p, (1 << 30) // B + 1, batch, o),       # B m > 2^30
                 lambda: ctx.trace_scene_batch_hits_ranged_into(d8.data_ptr(), -5, batch, o)]
        plan = ctx.last_plan()
        for call in calls:
            with pytest.raises(R.RayError):
                call()
        assert ctx.last_plan() == plan
        n0 = ctx.launch_count()
        ctx.trace_scene_batch_hits_into(p, 0, batch, None)                 # m == 0 does nothing
        ctx.trace_scene_batch_multi_hits_ranged_into(None, 0, batch, 3, None)
        rgb = torch.full((B, m, 3), 7.0, device="cuda")
        seg = torch.full((B, m), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.trace_scene_batch_paths_into(p, m, batch, rgb.data_ptr(), seg.data_ptr(), max_depth=0)
        ctx.sync()
        assert ctx.launch_count() == n0 and (_np(rgb) == 0).all() and (_np(seg) == 0).all()
        ctx.set_shard(0, 2)   # ignored: rays are not tiles
        for kind, rays, kw in cases(d6, d8, 4, (0.0, 1e9), 50)[:4]:
            n0 = ctx.launch_count()
            assert_same(run_batch(ctx, batch, kind, rays, **kw), want[kind], f"{kind} after the errors")
            assert ctx.launch_count() - n0 == 1 and ctx.last_render_ms() > 0
        ctx.set_shard(0, 1)
        hits = ctx.trace_scene_batch_hits(batch, d6)
        assert hits["t"].shape == (B, m) and hits["p"].shape == (B, m, 3)
        assert hits_differ(_np(torch.cat([hits["t"][..., None], hits["sphere"].view(torch.float32)[..., None], hits["p"],
                                          hits["normal"]], -1)).reshape(-1, 8), want["hits"]["records"].reshape(-1, 8)) == 0
        rgb, seg = ctx.trace_scene_batch_paths(batch, d6)
        assert bits_differ(_np(rgb), want["paths"]["rgb"]) == 0 and (_np(seg) == want["paths"]["segments"]).all()
        assert (_np(ctx.trace_scene_batch_occluded(batch, d6)).view(np.uint8) == want["occluded"]["occluded"]).all()
        mh = ctx.trace_scene_batch_multi_hits(batch, d6, 4)
        assert mh["t"].shape == (B, m, 4) and (_np(mh["count"]) == want["multi_hits"]["counts"]).all()
