"""The warp-queue kernel on every staging plan it launches, bit for bit against the CPU oracle.

launch_warpqueue picks one of its template instantiations at run time from the launch plan: the query kind, K (rays in
flight per warp / 32), spread samples, the packet walk, per-ray intervals, and how much of the scene sits in shared
memory: a prefix of the nodes ("partial"), every node with the spheres read from global memory ("nodes"), or every node
and every sphere record ("whole").  Which case a scene reaches depends on its size and the plan, so every case here
first checks through Context.last_plan() that the launch it was written for is the one that ran, and each kind group
ends by checking that its matrix launched every instantiation that is reachable.  Frames are compared with
oracle/pyoracle.py, ray queries with tests/ray_query_oracle.py.
"""
import numpy as np
import pytest

import ray_query_oracle as Q
from oracle import pyoracle as O
from ray_query_cases import _dev, _np, _torch, bits_differ, hits_differ, random_rays

H, W = 48, 64
SENTINEL = 0x7FA5A5A5
STAGING = {(0, 0): "partial", (1, 0): "nodes", (1, 1): "whole"}
PIXEL_KINDS = ("pixels", "accumulate", "views")
RAY_KINDS = ("closest", "anyhit", "multihit")
FORCED_PLANS = [dict(wq_k=1, wq_warps=32), dict(wq_k=2, wq_warps=16)]
MULTI_K = 4
CHUNK = 2048          # stage_scene copies 32 KB pieces: 512 nodes or 2048 sphere records


def staging(plan):
    return STAGING[(plan["all_nodes"], plan["spheres"])]


def variant(plan):
    """The axes launch_warpqueue dispatches on: (kind, ranged, K, spread, packet walk, staging case)."""
    return (plan["query"], bool(plan["ranged"]), plan["k"], bool(plan["spread"]), plan["packet"] > 0, staging(plan))


def reachable_pixel_variants():
    return {(q, False, k, sp, pk, st) for q in PIXEL_KINDS for k in (1, 2) for sp in (False, True) for pk in (False, True)
            for st in STAGING.values()}


def reachable_ray_variants():
    return {(q, rg, k, False, False, st) for q in RAY_KINDS for rg in (False, True) for k in (1, 2) for st in STAGING.values()}


def expect(plan, what, **want):
    got = {k: plan[k] for k in want}
    assert got == want, f"{what}: expected {want}, launched {plan}"


# ------------------------------------------------------------------------------------------ scenes and rays


def dense_scene(n, seed=7):
    """n random spheres in a cube small enough that most camera rays and random rays meet several of them."""
    rng = np.random.default_rng(seed)
    side = 2.2 * n ** (1 / 3)
    s = np.empty((n, 7), np.float32)
    s[:, 0:3] = rng.uniform(-side / 2, side / 2, (n, 3))
    s[:, 3:6] = rng.uniform(0.2, 0.95, (n, 3))
    s[:, 6] = rng.uniform(0.4, 1.2, n)
    cam = np.float32([0.35 * side, 0.45 * side, 1.7 * side, 0, 0, 0, 50])
    return s, cam


def second_camera(cam):
    c = cam.copy()
    c[0:3] = [-c[2] * 0.8, c[1] * 0.5, c[2] * 0.9]
    return c


class Case:
    """A dense scene of n spheres on the GPU side and in the oracle, and its packed tree (BFS node order)."""

    def __init__(self, R, n, seed=7):
        self.n, self.n_inner = n, n - 1
        self.spheres, self.cam = dense_scene(n, seed)
        self.oracle = Q.prepare_custom(self.spheres, self.cam, H, W)
        with R.Context(device=0) as ctx:
            pr = self.prepare(ctx)
            nodes = pr.packed()["nodes"]
            self.perm = pr.dump()["perm"]
            pr.free()
        self.left = nodes[:, 3].view(np.int32).copy()
        self.right = nodes[:, 7].view(np.int32).copy()

    def prepare(self, ctx, h=H, w=W):
        return ctx.prepare_scene(h, w, ctx.scene_from_arrays(self.spheres, self.cam))

    def leaves_below(self, node):
        out, stack = [], [node]
        while stack:
            c = stack.pop()
            for ch in (self.left[c], self.right[c]):
                if ch < 0:
                    out.append(int(~ch))
                else:
                    stack.append(int(ch))
        return sorted(out)

    def aimed_rays(self, nodes=(), leaves=(), seed=0):
        """Rays from outside the scene's box toward the centres of up to four leaves below each packed node of `nodes`
        and of each Morton-sorted leaf of `leaves` (indices past the tree are skipped).  Returns (rays, the caller's
        index of each ray's target sphere, the target node or leaf each ray belongs to)."""
        targets, group = [], []
        for i in nodes:
            if 0 <= i < self.n_inner:
                below = self.leaves_below(i)
                pick = sorted({below[0], below[len(below) // 3], below[2 * len(below) // 3], below[-1]})
                targets += pick
                group += [f"node {i}"] * len(pick)
        for j in leaves:
            if 0 <= j < self.n:
                targets.append(j)
                group.append(f"leaf {j}")
        idx = self.perm[np.asarray(targets, np.int64)]
        c = self.spheres[idx, 0:3]
        lo = (self.spheres[:, :3] - self.spheres[:, 6:7]).min(0)
        hi = (self.spheres[:, :3] + self.spheres[:, 6:7]).max(0)
        rng = np.random.default_rng(seed)
        u = rng.standard_normal((len(idx), 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        o = c + u * float(np.linalg.norm(hi - lo))
        return np.ascontiguousarray(np.concatenate([o, -u], 1), np.float32), idx, np.asarray(group)

    def rays(self, nodes=(), leaves=(), seed=0):
        """Random rays plus the aimed rays, after checking in the oracle's multi-hit lists that every target node's
        subtree and every target leaf is reached by some aimed ray (a ray that accepts a sphere below a node walked it)."""
        aimed, idx, group = self.aimed_rays(nodes, leaves, seed)
        if len(idx):
            rec, _ = self.oracle.trace_multi_hits(aimed, 64)
            reached = (rec[:, :, 1].view(np.int32) == idx[:, None]).any(1)
            missed = sorted(set(group) - set(group[reached]))
            assert not missed, f"no aimed ray reaches {missed}"
        rays = np.concatenate([random_rays(self.spheres, 768, seed + 1), aimed])
        rng = np.random.default_rng(seed + 2)
        t_min = rng.choice(np.float32([0.0, 0.1, 1.0, 2.5]), len(rays))
        t_max = rng.choice(np.float32([1e9, 6.0, 40.0]), len(rays))
        rays8 = np.concatenate([rays[:, :3], t_min[:, None], rays[:, 3:], t_max[:, None]], 1).astype(np.float32)
        return rays, rays8


# ------------------------------------------------------------------------------------------ GPU runs


def gpu_frame(ctx, pr, spp, h=H, w=W):
    torch = _torch()
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb), ctx.last_plan()


def oracle_frame(spheres, cam, spp, h=H, w=W):
    pix, rgb, _ = O.Scene.custom(spheres, cam).prepare(h, w).render(h, w, spp, want_rgb=True)
    return pix, rgb


def check_frame(got, want, what):
    assert (got[0] == want[0]).all(), f"{what}: {(got[0] != want[0]).sum()} pixels differ"
    assert bits_differ(got[1], want[1]) == 0, f"{what}: float framebuffer"


def ray_queries(ctx, pr, case, rays, rays8, what):
    """Every ray query (per-call and ranged) against the oracle; returns the plans they launched, by query."""
    torch = _torch()
    o, n, k = case.oracle, len(rays), MULTI_K
    d, d8 = _dev(rays), _dev(rays8)
    hits = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    multi = torch.empty((n, k, 8), dtype=torch.float32, device="cuda")
    counts = torch.empty((n,), dtype=torch.int32, device="cuda")
    occ = torch.empty((n,), dtype=torch.bool, device="cuda")
    torch.cuda.synchronize()
    plans = {}

    def run(name, call, check):
        call()
        ctx.sync()
        plans[name] = ctx.last_plan()
        check()

    run("hits", lambda: ctx.trace_hits_into(d.data_ptr(), n, pr, hits.data_ptr(), t_min=0.1, t_max=1e9),
        lambda: _eq(hits_differ(_np(hits), o.trace_hits(rays, 0.1, 1e9)), f"{what}: trace_hits"))

    def paths():
        rgb, seg = ctx.trace_paths(pr, d)
        plans["paths"] = ctx.last_plan()
        want_rgb, want_seg = o.trace_paths(rays)
        _eq(bits_differ(_np(rgb), want_rgb) + int((_np(seg) != want_seg).sum()), f"{what}: trace_paths")
    paths()
    run("occluded", lambda: ctx.trace_occluded_into(d.data_ptr(), n, pr, occ.data_ptr(), t_min=0.1, t_max=1e9),
        lambda: _eq(int((_np(occ) != o.trace_occluded(rays, 0.1, 1e9)).sum()), f"{what}: trace_occluded"))

    def check_multi(want):
        _eq(hits_differ(_np(multi).reshape(-1, 8), want[0].reshape(-1, 8)) + int((_np(counts) != want[1]).sum()),
            f"{what}: multi-hit")
    run("multi", lambda: ctx.trace_multi_hits_into(d.data_ptr(), n, pr, k, multi.data_ptr(), counts.data_ptr()),
        lambda: check_multi(o.trace_multi_hits(rays, k)))
    run("hits_ranged", lambda: ctx.trace_hits_ranged_into(d8.data_ptr(), n, pr, hits.data_ptr()),
        lambda: _eq(hits_differ(_np(hits), o.trace_hits_ranged(rays8)), f"{what}: trace_hits_ranged"))
    run("occluded_ranged", lambda: ctx.trace_occluded_ranged_into(d8.data_ptr(), n, pr, occ.data_ptr()),
        lambda: _eq(int((_np(occ) != o.trace_occluded_ranged(rays8)).sum()), f"{what}: trace_occluded_ranged"))
    run("multi_ranged", lambda: ctx.trace_multi_hits_ranged_into(d8.data_ptr(), n, pr, k, multi.data_ptr(), counts.data_ptr()),
        lambda: check_multi(o.trace_multi_hits_ranged(rays8, k)))
    return plans


RAY_QUERY_KINDS = {"hits": ("closest", 0), "paths": ("closest", 0), "occluded": ("anyhit", 0), "multi": ("multihit", 0),
                   "hits_ranged": ("closest", 1), "occluded_ranged": ("anyhit", 1), "multi_ranged": ("multihit", 1)}


def _eq(bad, what):
    assert bad == 0, f"{what}: {bad} values differ"


def check_ray_plans(plans, what, **want):
    for name, plan in plans.items():
        q, ranged = RAY_QUERY_KINDS[name]
        expect(plan, f"{what} {name}", query=q, ranged=ranged, spread=0, packet=0, **want)


# ------------------------------------------------------------------------------------------ a. forced boundaries


@pytest.fixture(scope="module")
def forced(R):
    """A scene that fits whole under every plan of FORCED_PLANS (sized from the staging budgets they report, at most 500
    spheres), its stage_cap points, and the oracle's frames, views and per-sample colours of it."""
    probe = Case(R, 500)
    budget = []
    for plan in FORCED_PLANS:
        for packet in (0, 8):
            with R.Context(device=0, wq_packet=packet, **plan) as ctx:
                pr = probe.prepare(ctx)
                for spp in (1, 3):
                    gpu_frame(ctx, pr, spp, 8, 8)
                    budget.append(ctx.last_plan()["stage_budget"])
    n = min(500, (min(budget) + 64) // 80)
    case = probe if n == 500 else Case(R, n)
    ni = n - 1
    caps = [("cap 0", 0, 4, 0), ("last node unstaged", 64 * (ni - 1), ni - 1, 0), ("nodes only", 64 * ni, ni, 0),
            ("one sphere short", 64 * ni + 16 * n - 16, ni, 0), ("whole", 64 * ni + 16 * n, ni, n), ("no cap", -1, ni, n)]
    cams = [case.cam, second_camera(case.cam)]
    frames = {spp: oracle_frame(case.spheres, case.cam, spp) for spp in (1, 2, 3)}
    views = {spp: [oracle_frame(case.spheres, c, spp) for c in cams] for spp in (1, 3)}
    colours = case.oracle.trace_paths(_camera_rays(R, case.oracle.camera(), 3))[0].reshape(H, W, 3, 3)
    sums = {2: colours[..., 0, :] + colours[..., 1, :]}
    sums[3] = sums[2] + colours[..., 2, :]
    return dict(case=case, caps=caps, cams=np.stack(cams), frames=frames, views=views, sums=sums, budgets=sorted(set(budget)))


def _camera_rays(R, camera, spp, h=H, w=W):
    return R.camera_rays(camera, h, w, spp).reshape(-1, 6)


@pytest.mark.gpu
def test_forced_boundaries_pixel_kinds(R, forced):
    """Frames, progressive chunks and views at every stage_cap point, K = 1 / 2, spread samples or not, with and without
    the packet walk: the exact staging split, and the oracle's frames."""
    torch = _torch()
    case, launched = forced["case"], set()
    for cap_name, cap, nodes, spheres in forced["caps"]:
        for plan in FORCED_PLANS:
            for packet in (0, 8):
                for spread in (1, 0):
                    what = f"{cap_name} (stage_cap {cap}), {plan}, wq_packet {packet}, wq_spread {spread}"
                    want = dict(kernel=R.KERNELS["warpqueue"], k=plan["wq_k"], warps=plan["wq_warps"], packet=packet,
                                smem_nodes=nodes, smem_spheres=spheres)
                    with R.Context(device=0, stage_cap=cap, wq_packet=packet, wq_spread=spread, **plan) as ctx:
                        pr = case.prepare(ctx)
                        for spp in ((1, 3) if spread else (3,)):
                            pix, rgb, p = gpu_frame(ctx, pr, spp)
                            expect(p, f"{what}, spp {spp}", query="pixels", spread=int(spread and spp > 1), **want)
                            check_frame((pix, rgb), forced["frames"][spp], f"{what}, spp {spp}")
                            launched.add(variant(p))
                        accum = torch.full((H, W, 3), float("nan"), dtype=torch.float32, device="cuda")
                        for a, b in ((0, 2), (2, 3)):
                            pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
                            p = ctx.last_plan()
                            expect(p, f"{what}, chunk [{a}, {b})", query="accumulate", spread=int(spread and b - a > 1), **want)
                            check_frame((_np(pix), _np(rgb)), forced["frames"][b], f"{what}, chunk [{a}, {b})")
                            assert bits_differ(_np(accum), forced["sums"][b]) == 0, f"{what}, chunk [{a}, {b}): sums"
                            launched.add(variant(p))
                        for spp in ((1, 3) if spread else (3,)):
                            pix, rgb = ctx.render_views(pr, forced["cams"], H, W, spp, want_rgb=True)
                            p = ctx.last_plan()
                            expect(p, f"{what}, views at spp {spp}", query="views", spread=int(spread and spp > 1), **want)
                            for v, want_v in enumerate(forced["views"][spp]):
                                check_frame((_np(pix[v]), _np(rgb[v])), want_v, f"{what}, view {v} at spp {spp}")
                            launched.add(variant(p))
    missing = reachable_pixel_variants() - launched
    assert not missing, f"pixel instantiations no case launched: {sorted(missing)}"
    assert launched == reachable_pixel_variants()


@pytest.mark.gpu
def test_forced_boundaries_ray_kinds(R, forced):
    """Every ray query, per-call and ranged, at every stage_cap point and K = 1 / 2, with rays aimed at the subtrees of
    the last staged node and the first unstaged one."""
    case, launched = forced["case"], set()
    for cap_name, cap, nodes, spheres in forced["caps"]:
        rays, rays8 = case.rays(nodes=(nodes - 1, nodes), seed=cap & 0xffff)
        for plan in FORCED_PLANS:
            what = f"{cap_name} (stage_cap {cap}), {plan}"
            with R.Context(device=0, stage_cap=cap, **plan) as ctx:
                plans = ray_queries(ctx, case.prepare(ctx), case, rays, rays8, what)
            check_ray_plans(plans, what, kernel=R.KERNELS["warpqueue"], k=plan["wq_k"], warps=plan["wq_warps"],
                            smem_nodes=nodes, smem_spheres=spheres)
            launched |= {variant(p) for p in plans.values()}
    missing = reachable_ray_variants() - launched
    assert not missing, f"ray-query instantiations no case launched: {sorted(missing)}"
    assert launched == reachable_ray_variants()


# ------------------------------------------------------------------------------------------ c. natural boundaries

NATURAL_PLANS = {"K1, 32 warps": dict(wq_k=1, wq_warps=32), "auto": {}, "K2, 16 warps": dict(wq_k=2, wq_warps=16),
                 "3 warps": dict(wq_warps=3)}


def _largest(pred, lo, hi):
    """The largest n in [lo, hi) with pred(n), for a pred that holds up to some n and not after it."""
    assert pred(lo) and not pred(hi), (lo, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(mid):
            lo = mid
        else:
            hi = mid
    return lo


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(NATURAL_PLANS))
def test_natural_boundaries(R, name):
    """stage_cap unset: the largest scene staged whole, the next one, the largest staged nodes only and the next one,
    found from the plans the library reports, each checked against the oracle with rays aimed at the staged / unstaged
    node boundary and, past 2048 staged records, at the second 32 KB piece of the staging copy."""
    plan_kw = NATURAL_PLANS[name]
    probes = {}
    with R.Context(device=0, **plan_kw) as ctx:
        def probe(n):
            if n not in probes:
                s, c = dense_scene(n)
                pr = ctx.prepare_scene(H, W, ctx.scene_from_arrays(s, c))
                d = _dev(random_rays(s, 64, 1))
                ctx.trace_hits(pr, d)
                probes[n] = ctx.last_plan()
                pr.free()
            return probes[n]
        n_whole = _largest(lambda n: staging(probe(n)) == "whole", 64, 6000)
        n_nodes = _largest(lambda n: probe(n)["all_nodes"] == 1, n_whole, 6000)
    budget = probes[n_whole]["stage_budget"]
    print(f"\nnatural staging boundaries, {name}: whole up to n = {n_whole} (budget {budget} B, K {probes[n_whole]['k']}, "
          f"{probes[n_whole]['warps']} warps), nodes only up to n = {n_nodes} "
          f"(budget {probes[n_nodes]['stage_budget']} B, K {probes[n_nodes]['k']}, {probes[n_nodes]['warps']} warps)")
    sizes = {n_whole: "whole", n_whole + 1: "nodes" if n_nodes > n_whole else "partial", n_nodes + 1: "partial"}
    if n_nodes > n_whole:
        sizes[n_nodes] = "nodes"
    else:
        # auto: the K = 1 plan it falls back to past the K = 2 whole-scene sizes leaves less room than K = 2 did, so
        # its scenes go from whole straight to partial
        assert name == "auto", f"{name}: no scene is staged nodes only"
    if name == "3 warps":
        assert n_whole > CHUNK, "the whole-scene case must run a second piece of sphere records"
    for n, want in sorted(sizes.items()):
        case = Case(R, n)
        with R.Context(device=0, **plan_kw) as ctx:
            pr = case.prepare(ctx, 32, 32)
            p = probes.get(n) or {}
            pix, rgb, fp = gpu_frame(ctx, pr, 1, 32, 32)
            what = f"{name}, n = {n}"
            assert staging(fp) == want, f"{what}: expected {want}, launched {fp}"
            check_frame((pix, rgb), oracle_frame(case.spheres, case.cam, 1, 32, 32), what)
            sn = fp["smem_nodes"]
            rays, rays8 = case.rays(nodes=(sn - 1, sn, CHUNK // 4 - 1, CHUNK // 4, CHUNK - 1, CHUNK),
                                    leaves=(CHUNK - 1, CHUNK, n - 1), seed=n)
            plans = ray_queries(ctx, pr, case, rays, rays8, what)
            check_ray_plans(plans, what, smem_nodes=sn, smem_spheres=fp["smem_spheres"], k=fp["k"], warps=fp["warps"])
            if p:
                assert (p["smem_nodes"], p["smem_spheres"]) == (sn, fp["smem_spheres"]), what


# ------------------------------------------------------------------------------------------ d. sample-count regimes


@pytest.mark.gpu
def test_sample_count_regimes(R):
    """Spread samples need a finished-sample buffer of SMs x warps x 8 x spp x 16 bytes within 1 GiB.  At 32 warps the
    last spp that spreads (1985 on a 132-SM H100) and the next one; at 3 warps spp 2500, which the frame's plan (made
    for 32 warps' buffer) does not expect to spread but the launch does, as a frame and as a progressive chunk."""
    torch = _torch()
    h, w = 4, 8
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    last = (1 << 30) // (sms * 32 * 8 * 16)
    sc = O.Scene.irreg()
    spheres, cam = sc.arrays()
    cases = [(dict(wq_k=1, wq_warps=32), last, 1), (dict(wq_k=1, wq_warps=32), last + 1, 0), (dict(wq_warps=3), 2500, 1)]
    for plan, spp, spread in cases:
        want = oracle_frame(spheres, cam, spp, h, w)
        with R.Context(device=0, **plan) as ctx:
            pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(spheres, cam))
            pix, rgb, p = gpu_frame(ctx, pr, spp, h, w)
            expect(p, f"{plan}, spp {spp}", query="pixels", spread=spread, warps=plan["wq_warps"])
            check_frame((pix, rgb), want, f"{plan}, spp {spp}")
            if plan["wq_warps"] == 3:
                accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
                pix, rgb = ctx.render_accumulate(pr, accum, 0, spp, want_rgb=True)
                expect(ctx.last_plan(), f"{plan}, chunk [0, {spp})", query="accumulate", spread=1, warps=3)
                check_frame((_np(pix), _np(rgb)), want, f"{plan}, chunk [0, {spp})")


# ------------------------------------------------------------------------------------------ e. the auto-K2 replan


@pytest.mark.gpu
def test_auto_k2_replans_with_k1(R):
    """wq_k = 0 plans K = 2 for a scene its queues leave whole; a stage_cap one sphere short of that makes the plan again
    with K = 1 (and 32 warps), which stages every node."""
    case = Case(R, 500)
    ni, n = case.n_inner, case.n
    rays, rays8 = case.rays(nodes=(ni - 1,), seed=3)
    with R.Context(device=0) as ctx:
        pr = case.prepare(ctx)
        frame = gpu_frame(ctx, pr, 1)
        expect(frame[2], "auto", k=2, all_nodes=1, spheres=1)
        check_ray_plans(ray_queries(ctx, pr, case, rays, rays8, "auto"), "auto", k=2, all_nodes=1, spheres=1)
    want = oracle_frame(case.spheres, case.cam, 1)
    with R.Context(device=0, stage_cap=64 * ni + 16 * n - 16) as ctx:
        pr = case.prepare(ctx)
        pix, rgb, p = gpu_frame(ctx, pr, 1)
        expect(p, "auto, one sphere short", k=1, warps=32, smem_nodes=ni, smem_spheres=0)
        check_frame((pix, rgb), want, "auto, one sphere short")
        plans = ray_queries(ctx, pr, case, rays, rays8, "auto, one sphere short")
        check_ray_plans(plans, "auto, one sphere short", k=1, warps=32, smem_nodes=ni, smem_spheres=0)
