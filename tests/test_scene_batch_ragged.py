"""Ragged scene batches (include/ray_b200.h "scene batches", ray_b200_scene_batch_new_ragged): B scenes of different
sphere counts n_b, packed back to back in one [N, 7] CUDA tensor.  Member b is bit for bit the prepared scene
prepare_scene_device makes of scene b's own records (its own refit sweeps and stale boxes included), frame b of a batch
render is render_into of member b, and every batch ray query answers as the member's, with spheres in [0, n_b).

On the CPU: the Python argument checks and the binding.  On the GPU: members against single builds on count mixes that
cross every refit-sweep step, skewed and large batches; uniform counts against new_device; frames, the float64 reference,
ray queries and every plan; updates that change the counts, ordering, memory and errors."""
import os
import re

import numpy as np
import pytest

import limit_scenes as LS
import ray_query_oracle as Q
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ
from test_input_ranges import ALL_SCENES, _builtin, assert_frame
from test_scene_batch import STAGING, assert_same_scene, frame, frames_of, random_batch
from test_scene_batch_rays import (PLAN_QUERY, assert_local_spheres, assert_same, batch_rays, cases, ranged, run_batch,
                                   run_oracle, run_single, scene_rays)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 24, 32
SYMBOLS = ["ray_b200_scene_batch_new_ragged", "ray_b200_scene_batch_update_ragged", "ray_b200_scene_batch_counts"]


# ------------------------------------------------------------------------------------------ batches


def pack(members):
    """(spheres [N, 7], cameras [B, 7], counts [B]) of a list of (spheres [n_b, 7], camera [7])"""
    s = np.ascontiguousarray(np.concatenate([np.asarray(m[0], np.float32) for m in members]), np.float32)
    cams = np.ascontiguousarray(np.stack([np.asarray(m[1], np.float32) for m in members]), np.float32)
    return s, cams, np.array([len(m[0]) for m in members], np.int64)


def random_ragged(counts, seed=1):
    """Random scenes of the given counts (random_batch's scenes, one seed each)"""
    members = []
    for b, n in enumerate(counts):
        s, c = random_batch(1, int(n), seed=seed * 7919 + b)
        members.append((s[0], c[0]))
    return pack(members)


def natural_members():
    """mixed_batch's members at their own sizes: rgbbox (stale boxes), irreg, every input-range scene, coincident
    centres, duplicates, a deep comb, a shallow random scene"""
    members = [_builtin("rgbbox"), _builtin("irreg")]
    members += [ALL_SCENES[name]() for name in sorted(ALL_SCENES)]
    s, c = _builtin("rgbbox")
    same = np.repeat(s[:1], 37, 0)
    same[:, 3:6] = np.linspace(0.1, 0.9, 37, dtype=np.float32)[:, None]
    members.append((same, c))
    members.append((np.concatenate([s[:50], s[:50]]), c))
    comb, _ = LS.comb_scene(300)
    members.append((comb, LS.COMB_CAM))
    r, rc = random_batch(1, 5, seed=5)
    members.append((r[0], rc[0]))
    assert all(len(m[0]) >= 2 for m in members)
    return pack(members)


def step_counts():
    """Counts on both sides of every trunc(log2f n) step from 2 to 2^17: 2^k - 1, 2^k, 2^k + 1"""
    return [2] + [n for k in range(2, 18) for n in ((1 << k) - 1, 1 << k, (1 << k) + 1)]


def offsets(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def members_of(s, counts):
    off = offsets(counts)
    return [s[off[b]:off[b + 1]] for b in range(len(counts))]


def check_members(R, ctx, batch, s, cams, counts, h, w, sample=None):
    """Every sampled member against prepare_scene_device of its records; returns the members' info"""
    B = len(counts)
    assert (batch.counts == counts).all() and batch.shape == (B, int(counts[0]) if (counts == counts[0]).all() else 0)
    parts = members_of(s, counts)
    infos = {}
    for b in (range(B) if sample is None else sample):
        m = batch.member(b)
        want = ctx.prepare_scene_device(h, w, _dev(parts[b]), cams[b])
        assert_same_scene(m, want, f"member {b} of {B} (n = {counts[b]})")
        infos[b] = m.info()
        m.free(); want.free()
    return infos


# ------------------------------------------------------------------------------------------ CPU


class NoContext:
    device = 0


class FakeBatch:
    shape = (3, 0)
    ctx = NoContext()


def test_python_argument_checks(R):
    torch = _torch()
    s, cams, counts = random_ragged([2, 5, 3])
    t = torch.from_numpy(s)
    bad_counts = {"1-d sequence": [None, [], [[2, 5, 3]], [2.0, 5.0, 3.0], np.float32([2, 5, 3]), [True, True, True], "253"],
                  "at least 2 spheres": [[2, 5, 1, 2], [0, 10], [-3, 13]],
                  "2\\^26": [[1 << 26, 2], [(1 << 26) + 1], [1 << 62, 2]]}
    for msg, cs in bad_counts.items():
        for c in cs:
            with pytest.raises(ValueError, match=msg):
                R.scene_batch_counts(0, t, c)
            if c is not None:   # (None: a uniform batch)
                with pytest.raises(ValueError, match=msg):
                    R.Context.prepare_scene_batch(NoContext(), 8, 8, t, cams, counts=c)
    for c in ([2, 5, 4], [2, 5], [12], torch.tensor([2, 5, 3]) + 1):   # the sum is not the rows
        with pytest.raises(ValueError, match="sum"):
            R.scene_batch_counts(0, t, c)
    for sp in (s, None, t.double(), t[:, :6], t[None], torch.empty((10, 7), device="meta")):
        with pytest.raises(ValueError):
            R.scene_batch_counts(0, sp, counts)
    with pytest.raises(ValueError, match="CUDA"):
        R.scene_batch_counts(0, t, counts)                                         # a host tensor
    for c in ([2, 8], [2, 2, 2, 4]):                                                # not the batch's B counts
        with pytest.raises(ValueError, match="batch's 3 counts"):
            R.scene_batch_counts(0, t, c, B=3)
        with pytest.raises(ValueError, match="batch's 3 counts"):
            R.SceneBatch.update(FakeBatch(), t, counts=c)
    if not torch.cuda.is_available():
        return
    d = _dev(s)
    B, c = R.scene_batch_counts(0, d, torch.tensor([2, 5, 3]))
    assert B == 3 and c.dtype == np.int64 and (c == [2, 5, 3]).all()
    for sp in (d.double(), d[::2], d.t().contiguous().t(), d[:, :6]):
        with pytest.raises(ValueError):
            R.scene_batch_counts(0, sp, counts)
    with pytest.raises(ValueError, match="cams"):
        R.Context.prepare_scene_batch(NoContext(), 8, 8, d, cams[:2], counts=[2, 5, 3])
    with pytest.raises(ValueError, match="host"):
        R.scene_batch_counts(0, d, torch.tensor([2, 5, 3], device="cuda"))
    with pytest.raises(ValueError):   # 2^20 frames of 64 x 32 tiles pass 2^25 tiles
        R.Context.prepare_scene_batch(NoContext(), 256, 256, torch.empty((1 << 21, 7), device="cuda"),
                                      np.zeros((1 << 20, 7)), counts=np.full(1 << 20, 2))


def test_header_declares_and_binding_binds_the_ragged_entry_points(R):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ray_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ray_b200_\w+)\s*\(", text))
    assert set(SYMBOLS) <= declared and set(SYMBOLS) <= set(R.declared_symbols())
    import ctypes
    lib = ctypes.CDLL(R.lib_path())
    assert all(hasattr(lib, f) for f in SYMBOLS)


# ------------------------------------------------------------------------------------------ GPU: build exactness


MIXES = {"small_and_large": lambda: random_ragged([2, 3, 1000, 2, 64], seed=1),
         "sweep_steps": lambda: random_ragged(step_counts(), seed=2),
         "natural": natural_members}


@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(MIXES))
def test_members_equal_single_builds(R, mix):
    """Every member, with its own refit sweeps: the natural and sweep-step mixes hold members with stale boxes whose sweep
    count is below the batch's largest, so a build that ran every scene to the largest count gives them other boxes."""
    h, w = 48, 64
    s, cams, counts = MIXES[mix]()
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        infos = check_members(R, ctx, batch, s, cams, counts, h, w)
        sweeps = {b: i["refit_sweeps"] for b, i in infos.items()}
        assert all(sweeps[b] == int(np.log2(np.float32(counts[b]))) + 2 for b in sweeps)
        short_stale = [b for b, i in infos.items() if i["stale_nodes"] > 0 and sweeps[b] < max(sweeps.values())]
        assert short_stale or mix == "small_and_large", "no member with stale boxes refits for fewer sweeps than the largest"
        if mix == "small_and_large":   # a few members also against the host builder and the oracle's boxes
            parts = members_of(s, counts)
            for b in (0, 1, 4):
                d = batch.member(b).dump()
                hl = R.host_lbvh(parts[b])
                for k in ("morton", "perm", "left", "right", "parent"):
                    np.testing.assert_array_equal(d[k], hl[k], err_msg=f"member {b} {k} vs host_lbvh")
                od = O.Scene.custom(parts[b], cams[b]).prepare(h, w).dump()
                np.testing.assert_array_equal(d["boxes"].view(np.uint32), od["boxes"].view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 7, 64, 1024])
def test_random_counts(R, B):
    rng = np.random.default_rng(B)
    counts = rng.integers(2, 700, B)
    s, cams, counts = random_ragged(counts, seed=B)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams, counts=counts)
        sample = range(B) if B <= 8 else sorted({0, 1, B // 3, B // 2, B - 2, B - 1, int(np.argmax(counts)), int(np.argmin(counts))})
        check_members(R, ctx, batch, s, cams, counts, H, W, sample)
        pix, rgb, plan = frames_of(ctx, batch, H, W, 2)
        assert plan["query"] == "scene_batch" and plan["n_inner"] == len(s) - B and plan["n_leaves"] == len(s)
        parts = members_of(s, counts)
        for b in sample:
            pr = ctx.prepare_scene_device(H, W, _dev(parts[b]), cams[b])
            assert_frame(pix[b], rgb[b], *frame(ctx, pr, H, W, 2), f"B={B} frame {b}")
            pr.free()


@pytest.mark.gpu
def test_skewed_batch(R):
    """One scene of 2^20 spheres next to 1023 scenes of 2: members, frames and hits of the large and the small scenes."""
    counts = np.array([1 << 20] + [2] * 1023, np.int64)
    s, cams, counts = random_ragged(counts, seed=3)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams, counts=counts)
        sample = [0, 1, 2, 511, 1023]
        check_members(R, ctx, batch, s, cams, counts, H, W, sample)
        pix, rgb, _ = frames_of(ctx, batch, H, W, 1)
        parts = members_of(s, counts)
        r6 = np.ascontiguousarray(np.stack([scene_rays(parts[b], 64, seed=b) for b in range(len(counts))]), np.float32)
        got = run_batch(ctx, batch, "hits", _dev(r6))
        for b in sample:
            pr = ctx.prepare_scene_device(H, W, _dev(parts[b]), cams[b])
            assert_frame(pix[b], rgb[b], *frame(ctx, pr, H, W, 1), f"frame {b}")
            assert_same({"records": got["records"][b]}, run_single(ctx, pr, "hits", _dev(r6[b])), f"hits of scene {b}")
            pr.free()
        assert_local_spheres({"records": got["records"][1:]}, 2, "the scenes of 2")


@pytest.mark.gpu
def test_uniform_counts_equal_new_device(R):
    """new_ragged with B equal counts and new_device(B, n) make the same batch: members, frames and queries."""
    B, n = 6, 150
    s, cams = random_batch(B, n, seed=17)
    with R.Context() as ctx:
        uni = ctx.prepare_scene_batch(H, W, _dev(s), cams)
        rag = ctx.prepare_scene_batch(H, W, _dev(s.reshape(-1, 7)), cams, counts=[n] * B)
        assert rag.shape == uni.shape == (B, n) and (rag.counts == n).all()
        for b in range(B):
            assert_same_scene(rag.member(b), uni.member(b), f"member {b}")
        for spp in (1, 4):
            a, b2 = frames_of(ctx, rag, H, W, spp), frames_of(ctx, uni, H, W, spp)
            assert (a[0] == b2[0]).all() and bits_differ(a[1], b2[1]) == 0 and a[2] == b2[2]
        r6 = batch_rays(s, 200, seed=4)
        d6, d8 = _dev(r6), _dev(ranged(r6, seed=4))
        for kind, rays, kw in cases(d6, d8, 5, (0.1, 1e9), 50):
            assert_same(run_batch(ctx, rag, kind, rays, **kw), run_batch(ctx, uni, kind, rays, **kw), f"{kind} {kw}")


# ------------------------------------------------------------------------------------------ GPU: frames


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,B,n", [(1, 1, 5, 64), (7, 13, 6, 100), (84, 84, 16, 64), (256, 256, 3, 1000), (1000, 1000, 2, 300)])
@pytest.mark.parametrize("spp", [1, 4, 16])
def test_frames_equal_member_and_independent_renders(R, h, w, B, n, spp):
    if h * w * spp > 1000 * 1000 * 4:
        pytest.skip("covered at fewer samples")
    counts = np.random.default_rng(h + B).integers(2, 2 * n, B)
    s, cams, counts = random_ragged(counts, seed=h + spp)
    parts = members_of(s, counts)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        pix, rgb, plan = frames_of(ctx, batch, h, w, spp)
        assert plan["query"] == "scene_batch"
        for b in range(B):
            m = batch.member(b)
            ind = ctx.prepare_scene_device(h, w, _dev(parts[b]), cams[b])
            assert_frame(pix[b], rgb[b], *frame(ctx, m, h, w, spp), f"frame {b} vs member")
            assert_frame(pix[b], rgb[b], *frame(ctx, ind, h, w, spp), f"frame {b} vs independent")
            if h * w <= 100:
                op, orgb, _ = O.Scene.custom(parts[b], cams[b]).prepare(h, w).render(h, w, spp, want_rgb=True)
                assert_frame(pix[b], rgb[b], op, orgb, f"frame {b} vs oracle")
            m.free(); ind.free()


@pytest.mark.gpu
def test_natural_members_frames(R):
    """mixed_batch's members at their own sizes, one frame each, against render_into of independent scenes"""
    h, w = 48, 64
    s, cams, counts = natural_members()
    parts = members_of(s, counts)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        pix, rgb, _ = frames_of(ctx, batch, h, w, 4)
        for b in range(len(counts)):
            pr = ctx.prepare_scene_device(h, w, _dev(parts[b]), cams[b])
            assert_frame(pix[b], rgb[b], *frame(ctx, pr, h, w, 4), f"frame {b}")
            pr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [("random", 0, "rgbbox", 0, "random", 1), ("rgbbox", 1, "random", 2, "rgbbox", 2)])
def test_float64_reference_judges_members(R, order):
    """Two ragged batches of the float64 reference's scene-batch members (random(3000) next to rgbbox): frames at spp 1 and
    3 and the one-segment queries of each member, judged against its own reference with the floors of its kind."""
    from test_f64_reference import assert_agrees, check_queries, judge_pixels, pick_pixels
    from test_f64_samples import BATCH_QUERIES, BATCH_SHAPE, FLOOR_BATCH, FLOOR_BATCH_RAYS, _batch, _batch_sources
    from test_f64_samples import batch_rays as f64_rays
    picks = list(zip(order[0::2], order[1::2]))
    members = [(_batch(kind)[0][i], _batch(kind)[1][i]) for kind, i in picks]
    s, cams, counts = pack(members)
    assert len(set(counts.tolist())) > 1
    h, w = BATCH_SHAPE
    j, i = pick_pixels(h, w, 200, 8)
    with R.Context(device=0) as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        for spp in (1, 3):
            pix, rgb = ctx.render_scene_batch(batch, h, w, spp, want_rgb=True)
            pix, rgb = _np(pix), _np(rgb)
            for b, (kind, k) in enumerate(picks):
                frac, bad, msg = judge_pixels(_batch(kind)[2][k], h, w, spp, j, i, pix[b][j, i], rgb[b][j, i])
                assert_agrees((frac, bad, f"member {b} ({kind} {k}): {msg}"), FLOOR_BATCH[kind, spp])
        for b, (kind, k) in enumerate(picks):
            rays = f64_rays(kind, k)
            src = _batch_sources(ctx, batch, b, len(picks))
            check_queries(_batch(kind)[2][k], rays, FLOOR_BATCH_RAYS[kind], *(src[q](rays) for q in BATCH_QUERIES))
        batch.free()


# ------------------------------------------------------------------------------------------ GPU: ray queries


def check_ragged(ctx, batch, s, counts, rays6, rays8, k, t, max_depth, refs, oracles=None, what=""):
    """Every entry point on a ragged batch against run_single on each scene's prepared scenes in refs (and the oracle)"""
    B = len(counts)
    d6, d8 = _dev(rays6), _dev(rays8)
    for kind, rays, kw in cases(d6, d8, k, t, max_depth):
        rg = rays.shape[2] == 8
        got = run_batch(ctx, batch, kind, rays, **kw)
        tag = f"{what} {kind}{' ranged' if rg else ''} {kw}"
        plan = ctx.last_plan()
        assert plan["query"] == PLAN_QUERY[kind] and plan["n_inner"] == len(s) - B and plan["n_leaves"] == len(s), (tag, plan)
        for b in range(B):
            mine = {key: v[b] for key, v in got.items()}
            assert_local_spheres(mine, int(counts[b]), f"{tag} scene {b}")
            for ref_name, prs in refs.items():
                assert_same(mine, run_single(ctx, prs[b], kind, rays[b], **kw), f"{tag} scene {b} vs {ref_name}")
            if oracles is not None:
                want = run_oracle(oracles[b], kind, (rays8 if rg else rays6)[b], **kw)
                assert_same(mine, want, f"{tag} scene {b} vs the oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["small_and_large", "natural"])
def test_every_query_equals_members_and_the_oracle(R, mix):
    s, cams, counts = MIXES[mix]()
    parts = members_of(s, counts)
    B = len(counts)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s), cams, counts=counts)
        refs = {"member": [batch.member(b) for b in range(B)],
                "independent": [ctx.prepare_scene_device(H, W, _dev(parts[b]), cams[b]) for b in range(B)]}
        oracles = [Q.prepare_custom(parts[b], cams[b], H, W) for b in range(B)]
        for i, (m, k, depth, t) in enumerate(((31, 7, 3, (0.1, 1e9)), (300, 64, 50, (0.0, 40.0)))):
            r6 = np.ascontiguousarray(np.stack([scene_rays(p, m, seed=50 * i + b) for b, p in enumerate(parts)]), np.float32)
            check_ragged(ctx, batch, s, counts, r6, ranged(r6, seed=i), k, t, depth, refs, oracles if i == 0 else None,
                         what=f"{mix} m={m}")


@pytest.mark.gpu
def test_every_plan_of_the_kinds(R):
    """Forced staging (partial, nodes, whole) x K = 1 / 2 for the render kind and the three ray kinds on a ragged batch:
    every answer equals the members'."""
    counts = np.array([2, 60, 17, 90, 3, 45, 128, 33], np.int64)
    s, cams, counts = random_ragged(counts, seed=11)
    parts = members_of(s, counts)
    B, N = len(counts), len(s)
    n_inner, n_leaves = N - B, N
    caps = {"partial": 64 * (n_inner // 3), "nodes": 64 * n_inner + 128, "whole": 64 * n_inner + 16 * n_leaves + 256}
    r6 = np.ascontiguousarray(np.stack([scene_rays(p, 200, seed=b) for b, p in enumerate(parts)]), np.float32)
    r8 = ranged(r6, seed=1)
    with R.Context() as ref:
        prs = [ref.prepare_scene_device(H, W, _dev(parts[b]), cams[b]) for b in range(B)]
        frames = {spp: [frame(ref, pr, H, W, spp) for pr in prs] for spp in (1, 4)}
        want = {}
        for kind, rays, kw in cases(_dev(r6), _dev(r8), 5, (0.1, 1e9), 50):
            want[kind, rays.shape[2] == 8] = [run_single(ref, prs[b], kind, rays[b], **kw) for b in range(B)]
    launched = set()
    for plan_kw in (dict(wq_k=1, wq_warps=32), dict(wq_k=2, wq_warps=16)):
        for stage, cap in caps.items():
            with R.Context(stage_cap=cap, wq_ncap=256, **plan_kw) as ctx:
                batch = ctx.prepare_scene_batch(H, W, _dev(s), cams, counts=counts)
                for spp in (1, 4):
                    pix, rgb, plan = frames_of(ctx, batch, H, W, spp)
                    what = f"{plan_kw} {stage} render spp {spp}"
                    assert plan["query"] == "scene_batch" and STAGING[(plan["all_nodes"], plan["spheres"])] == stage, (what, plan)
                    assert plan["k"] == plan_kw["wq_k"], (what, plan)
                    launched.add((plan["k"], stage, "scene_batch"))
                    for b in range(B):
                        assert_frame(pix[b], rgb[b], *frames[spp][b], f"{what} frame {b}")
                for kind, rays, kw in cases(_dev(r6), _dev(r8), 5, (0.1, 1e9), 50):
                    rg = rays.shape[2] == 8
                    got = run_batch(ctx, batch, kind, rays, **kw)
                    plan = ctx.last_plan()
                    what = f"{plan_kw} {stage} {kind} ranged={rg}"
                    assert plan["query"] == PLAN_QUERY[kind] and STAGING[(plan["all_nodes"], plan["spheres"])] == stage, (what, plan)
                    assert plan["k"] == plan_kw["wq_k"], (what, plan)
                    launched.add((plan["k"], stage, plan["query"]))
                    for b in range(B):
                        assert_same({key: v[b] for key, v in got.items()}, want[kind, rg][b], f"{what} scene {b}")
    reachable = {(k, st, q) for k in (1, 2) for st in STAGING.values()
                 for q in ("scene_batch", "scene_batch_closest", "scene_batch_anyhit", "scene_batch_multihit")}
    assert launched == reachable, reachable - launched


# ------------------------------------------------------------------------------------------ GPU: updates and ordering


@pytest.mark.gpu
def test_update_changes_the_counts(R):
    """An update that grows one member, shrinks another and keeps the rest: every member and frame is the new scene's;
    a uniform update of the unequal batch is refused and changes nothing; an update to equal counts makes it uniform."""
    counts0 = np.array([40, 300, 2, 77], np.int64)
    s0, cams, _ = random_ragged(counts0, seed=5)
    counts1 = np.array([40, 20, 900, 77], np.int64)
    s1, _, _ = random_ragged(counts1, seed=6)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(H, W, _dev(s0), cams, counts=counts0)
        batch.update(_dev(s1), counts=counts1)
        check_members(R, ctx, batch, s1, cams, counts1, H, W)
        fresh = ctx.prepare_scene_batch(H, W, _dev(s1), cams, counts=counts1)
        a, b2 = frames_of(ctx, batch, H, W, 4), frames_of(ctx, fresh, H, W, 4)
        assert (a[0] == b2[0]).all() and bits_differ(a[1], b2[1]) == 0
        with pytest.raises(R.RayError):
            batch.update_from_ptr(_dev(s1).data_ptr())                     # the uniform update of an unequal batch
        with pytest.raises(ValueError):
            batch.update(_dev(s1), counts=counts1[:3])
        with pytest.raises(ValueError):
            batch.update(_dev(np.zeros((4, 2, 7), np.float32)))
        assert (frames_of(ctx, batch, H, W, 4)[0] == a[0]).all() and (batch.counts == counts1).all()
        u, ucams = random_batch(4, 50, seed=7)
        batch.update(_dev(u.reshape(-1, 7)), ucams, counts=[50] * 4)
        assert batch.shape == (4, 50)
        batch.update(_dev(u))                                              # now uniform: the uniform update applies
        check_members(R, ctx, batch, u.reshape(-1, 7), ucams, np.full(4, 50), H, W)
        batch.free(); fresh.free()


@pytest.mark.gpu
def test_frames_and_queries_in_flight_read_the_old_trees(R):
    torch = _torch()
    h, w = 256, 256
    counts0 = np.array([2000, 30, 900, 5], np.int64)
    counts1 = np.array([100, 3000, 7, 600], np.int64)
    s0, cams, _ = random_ragged(counts0, seed=8)
    s1, _, _ = random_ragged(counts1, seed=9)
    r6 = np.ascontiguousarray(np.stack([scene_rays(p, 500, seed=b) for b, p in enumerate(members_of(s0, counts0))]), np.float32)
    with R.Context() as ctx:
        old = ctx.prepare_scene_batch(h, w, _dev(s0), cams, counts=counts0)
        new = ctx.prepare_scene_batch(h, w, _dev(s1), cams, counts=counts1)
        old_want, new_want = frames_of(ctx, old, h, w, 16)[0], frames_of(ctx, new, h, w, 16)[0]
        old_hits, new_hits = run_batch(ctx, old, "hits", _dev(r6)), run_batch(ctx, new, "hits", _dev(r6))
        assert (old_want != new_want).any()
        batch = ctx.prepare_scene_batch(h, w, _dev(s0), cams, counts=counts0)
        a = torch.empty((4, h, w), dtype=torch.int32, device="cuda")
        b2 = torch.empty((4, h, w), dtype=torch.int32, device="cuda")
        ha = torch.empty((4, 500, 8), dtype=torch.float32, device="cuda")
        hb = torch.empty((4, 500, 8), dtype=torch.float32, device="cuda")
        d6 = _dev(r6)
        torch.cuda.synchronize()
        ctx.render_scene_batch_into(batch, h, w, 16, a.data_ptr())
        ctx.trace_scene_batch_hits_into(d6.data_ptr(), 500, batch, ha.data_ptr())
        batch.update(_dev(s1), counts=counts1)
        ctx.render_scene_batch_into(batch, h, w, 16, b2.data_ptr())
        ctx.trace_scene_batch_hits_into(d6.data_ptr(), 500, batch, hb.data_ptr())
        batch.free()                      # with the second render and query possibly still running
        ctx.sync()
        assert (_np(a) == old_want).all() and (_np(b2) == new_want).all()
        assert bits_differ(_np(ha), old_hits["records"]) == 0 and bits_differ(_np(hb), new_hits["records"]) == 0


# ------------------------------------------------------------------------------------------ GPU: limits and memory


@pytest.mark.gpu
def test_largest_skewed_batch(R):
    """N = 2^26 with one scene of 2^25 spheres and 2^24 scenes of 2: a sample of members against their own builds."""
    torch = _torch()
    B = (1 << 24) + 1
    counts = np.full(B, 2, np.int64)
    counts[0] = 1 << 25
    gen = torch.Generator(device="cuda").manual_seed(3)
    s = torch.rand((1 << 26, 7), device="cuda", generator=gen)
    s[:, 0:3] *= 40.0
    s[:, 6] = s[:, 6] * 0.8 + 0.2
    cams = np.tile(np.float32([20, 30, 120, 20, 20, 20, 50]), (B, 1))
    off = offsets(counts)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(4, 8, s, cams, counts=counts)
        for b in (0, 1, B // 2, B - 1):
            m = batch.member(b)
            want = ctx.prepare_scene_device(4, 8, s[off[b]:off[b + 1]].contiguous(), cams[b])
            assert_same_scene(m, want, f"member {b}")
            m.free(); want.free()
        pix = ctx.render_scene_batch(batch, 4, 8)
        for b in (0, B - 1):
            want = ctx.prepare_scene_device(4, 8, s[off[b]:off[b + 1]].contiguous(), cams[b])
            assert (_np(pix[b]) == frame(ctx, want, 4, 8, 1)[0]).all()
            want.free()


@pytest.mark.gpu
def test_most_tiles(R):
    """B x tiles(h, w) = 2^25: 2^15 ragged scenes of 2 to 9 spheres, 1024 tiles each"""
    torch = _torch()
    h, w, B = 128, 256, 1 << 15
    counts = np.random.default_rng(1).integers(2, 10, B)
    s, cams, counts = random_ragged(counts, seed=12)
    parts = members_of(s, counts)
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        pix = torch.empty((B, h, w), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.render_scene_batch_into(batch, h, w, 1, pix.data_ptr())
        ctx.sync()
        for b in (0, 1, B // 2, B - 1):
            pr = ctx.prepare_scene_device(h, w, _dev(parts[b]), cams[b])
            assert (_np(pix[b]) == frame(ctx, pr, h, w, 1)[0]).all(), b
            pr.free()
        with pytest.raises(R.RayError):
            ctx.prepare_scene_batch_ragged_from_ptr(h, w + 8, _dev(s).data_ptr(), counts, cams)


@pytest.mark.gpu
def test_guarded_outputs_and_untouched_inputs(R):
    torch = _torch()
    h, w = 13, 21
    counts = np.array([40, 3, 17], np.int64)
    s, cams, counts = random_ragged(counts, seed=5)
    B, G = len(counts), 4096
    with R.Context() as ctx:
        t = _dev(s)
        before, cams_before, counts_before = _np(t).copy(), cams.copy(), counts.copy()
        batch = ctx.prepare_scene_batch(h, w, t, cams, counts=counts)
        want = frames_of(ctx, batch, h, w, 4)
        for fill in (0x00, 0xFF):
            guard = np.int32(fill * 0x01010101 - (1 << 32 if fill else 0))
            pix = torch.full((2 * G + B * h * w,), int(guard), dtype=torch.int32, device="cuda")
            rgb = torch.full((2 * G + B * h * w * 3,), int(guard), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.render_scene_batch_into(batch, h, w, 4, pix[G:].data_ptr(), rgb[G:].data_ptr())
            ctx.sync()
            p, r = _np(pix), _np(rgb)
            assert (p[:G] == guard).all() and (p[G + B * h * w:] == guard).all(), fill
            assert (r[:G] == guard).all() and (r[G + B * h * w * 3:] == guard).all(), fill
            assert (p[G:G + B * h * w].reshape(B, h, w) == want[0]).all()
            assert bits_differ(r[G:G + B * h * w * 3].view(np.float32).reshape(B, h, w, 3), want[1]) == 0
        batch.update(t, counts=counts)
        ctx.sync()
        assert (_np(t).view(np.uint32) == before.view(np.uint32)).all() and (cams == cams_before).all()
        assert (counts == counts_before).all()


@pytest.mark.gpu
@pytest.mark.parametrize("poison", [0x00, 0xFF, 0x7F])
def test_outputs_do_not_depend_on_pool_contents(R, poison):
    from test_memory_contract import Driver
    torch = _torch()
    h, w = 48, 64
    counts = np.array([300, 2, 51, 1000, 7], np.int64)
    s, cams, counts = random_ragged(counts, seed=13)
    with R.Context() as ref:
        want = frames_of(ref, ref.prepare_scene_batch(h, w, _dev(s), cams, counts=counts), h, w, 4)
    drv = Driver(0)
    st = torch.cuda.Stream()
    with R.Context() as ctx, torch.cuda.stream(st):
        ctx.set_stream(st.cuda_stream)
        t = _dev(s)
        st.synchronize()
        drv.poison_pool(st.cuda_stream, poison)
        batch = ctx.prepare_scene_batch(h, w, t, cams, counts=counts)
        drv.poison_pool(st.cuda_stream, poison)
        batch.update(t, counts=counts)
        drv.poison_pool(st.cuda_stream, poison)
        got = frames_of(ctx, batch, h, w, 4)
        m = batch.member(3)
        drv.poison_pool(st.cuda_stream, poison)
        assert (frame(ctx, m, h, w, 4)[0] == want[0][3]).all()
        batch.free(); m.free()
        ctx.set_stream(None)
    assert (got[0] == want[0]).all() and bits_differ(got[1], want[1]) == 0


@pytest.mark.gpu
def test_errors_leave_the_batch_and_context_usable(R):
    h, w = 16, 16
    counts = np.array([20, 3, 9], np.int64)
    s, cams, counts = random_ragged(counts, seed=2)
    t = _dev(s)
    p = t.data_ptr()
    with R.Context() as ctx:
        batch = ctx.prepare_scene_batch(h, w, t, cams, counts=counts)
        want = frames_of(ctx, batch, h, w, 1)[0]
        lib, hd = ctx.lib, ctx.handle
        c = np.ascontiguousarray(cams)
        import ctypes as C
        out = C.c_void_p(None)
        for bad in ([20, 3, 1], [20, 0, 9], [1 << 26, 2, 2], [-5, 3, 9]):
            cc = np.ascontiguousarray(bad, np.int64)
            with pytest.raises(R.RayError):
                ctx._check(lib.ray_b200_scene_batch_new_ragged(hd, C.byref(out), h, w, p, 3, cc.ctypes.data, c.ctypes.data))
            with pytest.raises(R.RayError):
                batch.update_ragged_from_ptr(p, cc)
        for call in (lambda: ctx._check(lib.ray_b200_scene_batch_new_ragged(hd, C.byref(out), h, w, p, 3, None, c.ctypes.data)),
                     lambda: ctx._check(lib.ray_b200_scene_batch_update_ragged(hd, batch.handle, p, None, None)),
                     lambda: ctx._check(lib.ray_b200_scene_batch_counts(hd, batch.handle, None)),
                     lambda: ctx.prepare_scene_batch_ragged_from_ptr(h, w, 0, counts, cams),
                     lambda: ctx.prepare_scene_batch_ragged_from_ptr(h, w, s.ctypes.data, counts, cams),   # host memory
                     lambda: ctx.prepare_scene_batch_ragged_from_ptr(0, w, p, counts, cams),
                     lambda: ctx.prepare_scene_batch_ragged_from_ptr(h, w, p, counts[:0], cams[:0]),
                     lambda: batch.update_ragged_from_ptr(s.ctypes.data, counts),
                     lambda: batch.member(3)):
            with pytest.raises(R.RayError):
                call()
        assert (frames_of(ctx, batch, h, w, 1)[0] == want).all() and (batch.counts == counts).all()
        check_members(R, ctx, batch, s, cams, counts, h, w)
        ctx.set_shard(0, 2)
        with pytest.raises(R.RayError):
            batch.update(t, counts=counts)
        ctx.set_shard(0, 1)
        assert (frames_of(ctx, batch, h, w, 1)[0] == want).all()


# ------------------------------------------------------------------------------------------ GPU: NaN centres


def nan_centre_scene(n, seed):
    """n random spheres whose last one has a NaN centre on x: a finite record whose box is [-inf, 0] (px = -3e38,
    r = 3e38), so its centre is -inf + inf"""
    s, c = random_batch(1, n, seed=seed)
    s = s[0].copy()
    s[-1, 0], s[-1, 6] = -3e38, 3e38
    return s, c[0]


def assert_host_build(R, ctx, pr, s, cam, h, w, what):
    """pr's LBVH against the host builder, its boxes against the oracle's, and its frame against the oracle's"""
    d, hl = pr.dump(), R.host_lbvh(s)
    for k in ("morton", "perm", "left", "right", "parent"):
        np.testing.assert_array_equal(d[k], hl[k], err_msg=f"{what}: {k} vs host_lbvh")
    op = O.Scene.custom(s, cam).prepare(h, w)
    np.testing.assert_array_equal(d["boxes"].view(np.uint32), op.dump()["boxes"].view(np.uint32), err_msg=f"{what}: boxes")
    assert (frame(ctx, pr, h, w, 1)[0] == op.render(h, w)[0]).all(), f"{what}: frame vs oracle"


@pytest.mark.gpu
def test_nan_centres_are_skipped_by_the_box_reduction(R):
    """The reference's centre box (bvh.fut:32-37, f32.minimum / maximum) skips NaN centres.  A NaN centre alone in the
    build's last, partial step of 32 spheres (a scene of 33), and alone for its scene in a step that crosses into the
    next scene (a ragged batch of 33 and 40), must leave the box, and so every Morton key, as the host builder makes it."""
    h, w = 24, 32
    single, cam = nan_centre_scene(33, 1)
    a, ca = nan_centre_scene(33, 2)
    b, cb = random_batch(1, 40, seed=3)
    s, cams, counts = pack([(a, ca), (b[0], cb[0]), (single, cam)])
    with R.Context() as ctx:
        pr = ctx.prepare_scene_device(h, w, _dev(single), cam)
        assert_host_build(R, ctx, pr, single, cam, h, w, "prepare_scene_device of 33")
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams, counts=counts)
        pix, rgb, _ = frames_of(ctx, batch, h, w, 1)
        for k, part in enumerate(members_of(s, counts)):
            m = batch.member(k)
            assert_host_build(R, ctx, m, part, cams[k], h, w, f"member {k}")
            assert_frame(pix[k], rgb[k], *frame(ctx, m, h, w, 1), f"frame {k}")
            m.free()
