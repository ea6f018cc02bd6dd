"""Frames and ray queries against tests/f64_reference.py, a float64 restatement of the reference's semantics that shares
no code with the oracle or the kernels.

The oracle and the kernels agree bit for bit, and the oracle is pinned by the reference only at the two 500 x 500
golden frames.  A misreading of ray.fut / bvh.fut or of include/ray_b200.h that both share (non-square frames, the spp
sample offsets, custom cameras and views, sphere indices in the caller's order, the interval quirks of objs_hit,
occlusion and multi-hit, max_depth, the stale boxes of the fixed-sweep refit) would pass every other test.  Here each
entry point's output is judged against the f64 reference: on the CPU through the oracle, on the GPU directly.

Only *judged* samples and rays are compared (f64_reference's margins and perturbation check), and each case asserts a
floor on its judged fraction, measured on the oracle and rounded down, so that no case passes by judging nothing.  The
mutation tests run the same comparison against deliberately wrong variants of the reference and assert that each is
rejected, which shows the comparison can tell.
"""
import functools

import numpy as np
import pytest

import f64_reference as F
import ray_query_oracle as Q
from limit_scenes import COMB_CAM, comb_query_rays, comb_scene
from oracle import pyoracle as O
from ray_query_cases import INTERVALS, SEGMENT, _dev, _np, _torch, light_above, random_rays, segment_rays
from test_input_ranges import PIXEL_SCENES

SHAPES = [(500, 500), (48, 160), (160, 48), (37, 53)]
SPPS = [1, 3, 16]
CUSTOM_SCENES = ["rgbbox_x255", "irreg_x255", "rgbbox_negative", "rgbbox_top_down"]
K = 4
RANDOM_N = 3000
COMB_M = 200

# Floors of the judged fractions.  A judged fraction depends on the reference and the inputs only, not on the output
# judged, so each was measured once (on the oracle's output, CPU) and rounded down; a case below its floor fails.
FLOOR_GOLDEN = {"rgbbox": 0.4, "irreg": 0.6}
FLOOR_FRAMES = {   # (scene, spp): the lowest over SHAPES
    ("rgbbox", 1): 0.3, ("rgbbox", 3): 0.15, ("rgbbox", 16): 0.02,
    ("irreg", 1): 0.55, ("irreg", 3): 0.5, ("irreg", 16): 0.5,
    ("random", 1): 0.8, ("random", 3): 0.65, ("random", 16): 0.55,
    ("rgbbox_x255", 1): 0.2, ("rgbbox_x255", 3): 0.05, ("rgbbox_negative", 1): 0.2, ("rgbbox_negative", 3): 0.05,
    ("irreg_x255", 1): 0.45, ("irreg_x255", 3): 0.45, ("rgbbox_top_down", 1): 0.95, ("rgbbox_top_down", 3): 0.95,
    ("comb", 1): 0.8, ("comb", 3): 0.8,
}
FLOOR_VIEWS = {1: 0.4, 3: 0.15}
FLOOR_SCRAMBLED = {"rgbbox": 0.4, "random": 0.9}
FLOOR_RAYS = {"rgbbox": 0.75, "irreg": 0.75, "random": 0.9, "comb": 0.6, "random1M": 0.25}   # every query kind
FLOOR_PATHS = {"rgbbox": 0.45, "irreg": 0.85, "random": 0.9}

# ------------------------------------------------------------------------------------------ scenes and references


@functools.lru_cache(maxsize=None)
def scene_arrays(name):
    """(spheres float32[n][7], cam7) of a named scene."""
    import raytracers_b200 as R
    if name in ("rgbbox", "irreg"):
        return R.host_scene(name)
    if name == "random":
        return R.host_scene("random", RANDOM_N, 1)
    if name == "comb":   # the comb of limit_scenes with small comb spheres, so the cluster decides the upper boxes
        s, first = comb_scene(COMB_M)
        s[:first - 1, 6] = 0.25
        return s, COMB_CAM
    return PIXEL_SCENES[name]()


@functools.lru_cache(maxsize=None)
def topology(name):
    import raytracers_b200 as R
    return R.host_lbvh(scene_arrays(name)[0])


@functools.lru_cache(maxsize=None)
def reference(name, mutant=None):
    s, c = scene_arrays(name)
    return F.Reference(s, topology(name), c, mutant)


def pick_pixels(h, w, count, seed):
    """Up to `count` distinct pixels (rows, columns) of an h x w frame, every pixel of a small frame."""
    k = np.arange(h * w) if h * w <= count else np.random.default_rng(seed).choice(h * w, count, replace=False)
    return k // w, k % w


def samples_for(spp):
    return max(40, 600 // spp)


# ------------------------------------------------------------------------------------------ comparisons


def judge_pixels(ref, h, w, spp, j, i, pix, rgb=None, cam7=None):
    """(judged fraction, disagreements on judged pixels, message) of pixels [len(j)] and float pixels [len(j)][3] of
    an h x w frame at spp against the f64 reference."""
    want, mean, err, judged = ref.pixels(h, w, j, i, spp, cam7)
    bad = judged & (np.asarray(pix) != want)
    if rgb is not None:
        rgb = np.asarray(rgb, np.float64)
        with np.errstate(invalid="ignore"):
            far = np.abs(rgb - mean) > (4 * err + 1e-6)[:, None] * np.maximum(1.0, np.abs(mean))
        bad |= judged & (far | (np.isnan(rgb) != np.isnan(mean))).any(1)
    frac = float(judged.mean())
    k = np.nonzero(bad)[0][:3]
    msg = (f"judged {frac:.3f} of {len(j)} pixels, {int(bad.sum())} judged pixels differ"
           + "".join(f"; ({j[x]}, {i[x]}) got {int(pix[x]):#x} want {int(want[x]):#x}" for x in k))
    return frac, int(bad.sum()), msg


def records_bad(ref, rays, rec, got):
    """Per record: the got record (float32[..., 8] of struct ray_b200_hit) is not the f64 one: another sphere, or t, p
    or normal further from it than f32 arithmetic on the ray's and the scene's magnitudes explains."""
    got = np.asarray(got, np.float32)
    r = np.asarray(rays, np.float64)[:, :6].reshape((len(rays),) + (1,) * (rec["t"].ndim - 1) + (6,))
    dn = np.maximum(np.sqrt(F._dot(r[..., 3:], r[..., 3:])), 1e-30)
    on = np.sqrt(F._dot(r[..., :3], r[..., :3]))
    t = np.abs(rec["t"])
    graze = 1e-6 * t / np.sqrt(np.maximum(rec["dm"], 1e-30))     # a root's f32 error near grazing
    tol_t = 1e-5 * (t + on / dn + 1.0) + graze
    tol_p = 1e-5 * (t * dn + on + 1.0) + graze * dn
    tol_n = tol_p / np.maximum(np.abs(ref.rad[np.maximum(rec["leaf"], 0)]), 1e-30) + 1e-5
    with np.errstate(invalid="ignore"):
        bad = got[..., 1].view(np.int32) != rec["sphere"]
        bad |= np.abs(got[..., 0] - rec["t"]) > tol_t
        bad |= (np.abs(got[..., 2:5] - rec["p"]) > tol_p[..., None]).any(-1)
        bad |= (np.abs(got[..., 5:8] - rec["normal"]) > tol_n[..., None]).any(-1)
    return bad


def _msg(kind, judged, bad):
    return f"{kind}: judged {judged.mean():.3f} of {len(judged)} rays, {int((bad & judged).sum())} judged rays differ"


def judge_hits(ref, rays, lo, hi, got):
    O, D = rays[:, :3].astype(np.float64), rays[:, 3:6].astype(np.float64)
    lo, hi = F.Reference._intervals(len(rays), lo, hi)
    rec = ref.closest(O, D, lo, hi)
    judged = rec["margin"] > F.TAU
    bad = records_bad(ref, rays, rec, got)
    return float(judged.mean()), int((bad & judged).sum()), _msg("hits", judged, bad)


def judge_occluded(ref, rays, lo, hi, got):
    occ, margin = ref.occluded(rays[:, :3].astype(np.float64), rays[:, 3:6].astype(np.float64), lo, hi)
    judged = margin > F.TAU
    bad = np.asarray(got, bool) != occ
    return float(judged.mean()), int((bad & judged).sum()), _msg("occluded", judged, bad)


def judge_multi(ref, rays, lo, hi, k, got, counts):
    rec, count, margin = ref.multi_hits(rays[:, :3].astype(np.float64), rays[:, 3:6].astype(np.float64), lo, hi, k)
    judged = margin > F.TAU
    bad = records_bad(ref, rays, rec, got).any(1) | (np.asarray(counts) != count)
    return float(judged.mean()), int((bad & judged).sum()), _msg(f"multi-hit k={k}", judged, bad)


def assert_agrees(result, floor):
    frac, bad, msg = result
    assert bad == 0, msg
    assert frac >= floor, f"judged fraction below its floor {floor}: {msg}"


# ------------------------------------------------------------------------------------------ rays


def surface_rays(spheres, n, seed, gap=0.05):
    """Rays that start `gap` outside a sphere and point at its centre: the near root lies between 0 and the search
    epsilon 0.1, so the closest hit is found at the far root and re-intersected on (t_min, t_best + 1)."""
    s = np.asarray(spheres, np.float32)
    rng = np.random.default_rng(seed)
    pick = s[rng.integers(0, len(s), n)]
    u = rng.standard_normal((n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = pick[:, :3] + (np.abs(pick[:, 6:7]) + gap) * u
    return np.ascontiguousarray(np.concatenate([o, -u], 1), np.float32)


def comb_rim_rays(n, seed):
    """Rays along the axes through the comb's cluster (radius 1 at the origin) that stay below -0.3 on the other two
    axes: they hit the cluster, but the comb's boxes above it, refitted short of the cluster's box, cull them."""
    rng = np.random.default_rng(seed)
    off = rng.uniform(-0.7, -0.3, (n, 2))
    axis = rng.integers(0, 3, n)
    o = np.zeros((n, 3))
    d = np.zeros((n, 3))
    for a in range(3):
        k = axis == a
        other = [x for x in range(3) if x != a]
        o[k, a], d[k, a] = -3.0, 1.0
        o[np.ix_(k, other)] = off[k]
    return np.ascontiguousarray(np.concatenate([o, d], 1), np.float32)


def comb_rays():
    return np.concatenate([comb_query_rays(600, 3), comb_rim_rays(300, 4)])


@functools.lru_cache(maxsize=None)
def query_rays(name, h=48, w=64):
    """Random rays, camera rays of an h x w frame, shadow rays from the camera rays' f64 hit points to a light above
    the scene, and rays starting just outside spheres: float32[n][6]."""
    import raytracers_b200 as R
    s, c = scene_arrays(name)
    rnd = random_rays(s, 600, 11)
    cam = R.camera_rays(R.host_camera(c, h, w), h, w).reshape(-1, 6)
    cam = cam[np.random.default_rng(12).choice(len(cam), min(len(cam), 600), replace=False)]
    hit = reference(name).closest(cam[:, :3].astype(np.float64), cam[:, 3:].astype(np.float64), 0.1, 1e9)
    shadow = segment_rays(hit["p"][hit["leaf"] >= 0].astype(np.float32), light_above(s))[:400]
    near = surface_rays(s, 300, 13)
    rays = np.concatenate([rnd, cam, shadow, near])
    return np.ascontiguousarray(rays, np.float32)


def ranged_intervals(n, seed):
    """Per-ray intervals: the per-call intervals, the segment interval, and a few the library answers as empty."""
    choices = INTERVALS + [SEGMENT, (float("nan"), 5.0), (-1.0, 5.0), (0.0, float("inf"))]
    k = np.random.default_rng(seed).integers(0, len(choices), n)
    iv = np.array(choices, np.float64)[k]
    return iv[:, 0].astype(np.float32), iv[:, 1].astype(np.float32)


def rays8(rays, lo, hi):
    r = np.asarray(rays, np.float32)
    return np.ascontiguousarray(np.concatenate([r[:, :3], lo[:, None], r[:, 3:], hi[:, None]], 1), np.float32)


def check_queries(ref, rays, floor, hits, occluded, multi, ranged_hits, ranged_occluded, ranged_multi):
    """Every query kind of one source (callables returning numpy) against the reference, at INTERVALS and with mixed
    per-ray intervals."""
    for lo, hi in INTERVALS:
        assert_agrees(judge_hits(ref, rays, lo, hi, hits(lo, hi)), floor)
        assert_agrees(judge_occluded(ref, rays, lo, hi, occluded(lo, hi)), floor)
        assert_agrees(judge_multi(ref, rays, lo, hi, K, *multi(lo, hi)), floor)
    lo, hi = ranged_intervals(len(rays), 5)
    r8 = rays8(rays, lo, hi)
    assert_agrees(judge_hits(ref, rays, lo, hi, ranged_hits(r8)), floor)
    assert_agrees(judge_occluded(ref, rays, lo, hi, ranged_occluded(r8)), floor)
    assert_agrees(judge_multi(ref, rays, lo, hi, K, *ranged_multi(r8)), floor)


# ------------------------------------------------------------------------------------------ CPU: the reference itself


@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_reference_reproduces_the_golden_pngs(golden, name):
    """The only real ground truth: on judged pixels, the f64 reference is the reference's own 500 x 500 frame."""
    want, _ = golden[f"{name}_500"]
    j, i = pick_pixels(500, 500, 1500, 1)
    assert_agrees(judge_pixels(reference(name), 500, 500, 1, j, i, want[j, i]), FLOOR_GOLDEN[name])


@pytest.mark.parametrize("name", ["rgbbox", "irreg", "random", "comb"])
def test_refitted_boxes_equal_host_lbvh(name):
    """The boxes refitted here from host_lbvh's topology alone equal its boxes bit for bit, and so does the number of
    stale boxes (those the fixed sweep count leaves short of the union of their children)."""
    topo, ref = topology(name), reference(name)
    assert ref.sweeps == topo["refit_sweeps"]
    assert np.array_equal(ref.boxes.view(np.uint32), topo["boxes"].view(np.uint32))
    assert int(ref.stale.sum()) == topo["stale_nodes"]
    if name == "rgbbox":
        assert topo["stale_nodes"] == 3
    if name == "comb":   # the refit stops short of the cluster's box on most comb levels
        assert int((ref.boxes != ref.fixpoint_boxes).any(1).sum()) >= 20


# ------------------------------------------------------------------------------------------ CPU: the oracle against it


@functools.lru_cache(maxsize=None)
def oracle_frame(name, h, w, spp):
    s, c = scene_arrays(name)
    pix, rgb, _ = O.Scene.custom(s, c).prepare(h, w).render(h, w, spp=spp, want_rgb=True)
    return pix, rgb


@pytest.mark.parametrize("spp", SPPS)
@pytest.mark.parametrize("h,w", SHAPES)
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_oracle_frames(name, h, w, spp):
    pix, rgb = oracle_frame(name, h, w, spp)
    j, i = pick_pixels(h, w, samples_for(spp), h * w + spp)
    assert_agrees(judge_pixels(reference(name), h, w, spp, j, i, pix[j, i], rgb[j, i]), FLOOR_FRAMES[name, spp])


@pytest.mark.parametrize("spp", [1, 3])
@pytest.mark.parametrize("name", CUSTOM_SCENES + ["comb"])
def test_oracle_frames_of_custom_scenes(name, spp):
    h, w = 37, 53
    pix, rgb = oracle_frame(name, h, w, spp)
    j, i = pick_pixels(h, w, samples_for(spp), 3)
    assert_agrees(judge_pixels(reference(name), h, w, spp, j, i, pix[j, i], rgb[j, i]), FLOOR_FRAMES[name, spp])


def _oracle_sources(o):
    return dict(hits=lambda rays: (lambda lo, hi: o.trace_hits(rays, lo, hi)),
                occluded=lambda rays: (lambda lo, hi: o.trace_occluded(rays, lo, hi)),
                multi=lambda rays: (lambda lo, hi: o.trace_multi_hits(rays, K, lo, hi)),
                ranged_hits=lambda rays: o.trace_hits_ranged,
                ranged_occluded=lambda rays: o.trace_occluded_ranged,
                ranged_multi=lambda rays: (lambda r8: o.trace_multi_hits_ranged(r8, K)))


@functools.lru_cache(maxsize=None)
def query_oracle(name):
    s, c = scene_arrays(name)
    return Q.prepare_custom(s, c, 48, 64)


@pytest.mark.parametrize("name", ["rgbbox", "irreg", "random", "comb"])
def test_ray_query_oracle(name):
    rays = comb_rays() if name == "comb" else query_rays(name)
    src = _oracle_sources(query_oracle(name))
    check_queries(reference(name), rays, FLOOR_RAYS[name], *(src[k](rays) for k in
                                           ("hits", "occluded", "multi", "ranged_hits", "ranged_occluded", "ranged_multi")))


@pytest.mark.parametrize("max_depth", [1, 3, 50])
@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_ray_query_oracle_paths(name, max_depth):
    rays = query_rays(name)[600:1200]
    rgb, seg = query_oracle(name).trace_paths(rays, max_depth)
    assert_agrees(judge_paths(reference(name), rays, max_depth, rgb, seg), FLOOR_PATHS[name])


def judge_paths(ref, rays, max_depth, rgb, seg):
    col, want_seg, _, err, judged = ref.judged_paths(rays[:, :3].astype(np.float64), rays[:, 3:].astype(np.float64),
                                                     max_depth)
    rgb = np.asarray(rgb, np.float64)
    with np.errstate(invalid="ignore"):
        far = np.abs(rgb - col) > (4 * err + 1e-6)[:, None] * np.maximum(1.0, np.abs(col))
    # NaN on one side only is a disagreement (a comparison with NaN is False, so `far` alone never sees it)
    bad = judged & ((np.asarray(seg) != want_seg) | (far | (np.isnan(rgb) != np.isnan(col))).any(1))
    return float(judged.mean()), int(bad.sum()), _msg(f"paths max_depth={max_depth}", judged, bad)


# ------------------------------------------------------------------------------------------ CPU: mutation tests


def _mutant_frame(mutant, name, h, w, spp):
    pix, rgb = oracle_frame(name, h, w, spp)
    j, i = pick_pixels(h, w, samples_for(spp), 7)
    return judge_pixels(reference(name, mutant), h, w, spp, j, i, pix[j, i], rgb[j, i])


def _mutant_hits(mutant, name, rays, lo):
    got = query_oracle(name).trace_hits(rays, lo, 1e9)
    return judge_hits(reference(name, mutant), rays, lo, 1e9, got)


def _sample_mutant(mutant):
    """A mutant of the per-sample, noise-estimate or G-buffer parts, rejected by test_f64_samples' case for it."""
    import test_f64_samples   # imported here: it imports this module
    return test_f64_samples.MUTANT_CASES[mutant](mutant)


MUTANT_CASES = {
    "offsets_in_f64": _sample_mutant, "welford_old_mean": _sample_mutant, "select_without_count": _sample_mutant,
    "gbuffer_depth_last_sample": _sample_mutant, "gbuffer_id_in_leaf_order": _sample_mutant,
    "gbuffer_miss_albedo_black": _sample_mutant,
    "aspect_h_over_w": lambda m: _mutant_frame(m, "rgbbox", 48, 160, 1),
    "v_from_j": lambda m: _mutant_frame(m, "irreg", 37, 53, 1),
    "offsets_s_plus_1": lambda m: _mutant_frame(m, "irreg", 37, 53, 3),
    "sky_from_x": lambda m: _mutant_frame(m, "irreg", 37, 53, 1),
    "no_stale_culling": lambda m: _mutant_hits(m, "comb", comb_rim_rays(300, 4), 0.0),
    "no_perm": lambda m: _mutant_hits(m, "rgbbox", query_rays("rgbbox"), 0.0),
    "reintersect_from_eps": lambda m: _mutant_hits(m, "rgbbox", surface_rays(scene_arrays("rgbbox")[0], 300, 13), 0.0),
}


def test_mutants_cover_the_list():
    assert set(MUTANT_CASES) == set(F.MUTANTS)


@pytest.mark.parametrize("mutant", list(F.MUTANTS))
def test_mutant_is_rejected(mutant):
    """The comparison, run against a deliberately wrong reference, must find judged disagreements."""
    frac, bad, msg = MUTANT_CASES[mutant](mutant)
    assert bad > 0, f"mutant {mutant} was not rejected: {msg}"


# ------------------------------------------------------------------------------------------ GPU: the product


def _gpu_prepared(ctx, name, h, w):
    s, c = scene_arrays(name)
    return ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))


@pytest.mark.gpu
@pytest.mark.parametrize("spp", SPPS)
@pytest.mark.parametrize("h,w", SHAPES)
@pytest.mark.parametrize("name", ["rgbbox", "irreg", "random"])
def test_render_into(R, name, h, w, spp):
    torch = _torch()
    with R.Context(device=0) as ctx:
        pr = _gpu_prepared(ctx, name, h, w)
        pix = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        rgb = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
        ctx.render_into(pix.data_ptr(), h, w, pr, spp, rgb.data_ptr())
        ctx.sync()
        pix, rgb = _np(pix), _np(rgb)
    j, i = pick_pixels(h, w, samples_for(spp), h * w + spp)
    assert_agrees(judge_pixels(reference(name), h, w, spp, j, i, pix[j, i], rgb[j, i]), FLOOR_FRAMES[name, spp])


VIEW_CAMS = np.float32([[0, 30, 30, 0, -1, -1, 75],
                        [25, 5, 28, 0, 0, -20, 40],
                        [-20, 20, 10, 5, -10, -25, 100],
                        [0, 0, 29, 0, 0, -30, 20]])


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 3])
def test_render_views(R, spp):
    """Four custom cameras (fov, look_at) of one prepared scene on a non-square frame, each judged with its own camera."""
    h, w = 40, 72
    with R.Context(device=0) as ctx:
        pr = _gpu_prepared(ctx, "rgbbox", h, w)
        pix, rgb = ctx.render_views(pr, VIEW_CAMS, h, w, spp, want_rgb=True)
        pix, rgb = _np(pix), _np(rgb)
    j, i = pick_pixels(h, w, samples_for(spp), 4)
    for v, cam in enumerate(VIEW_CAMS):
        frac, bad, msg = judge_pixels(reference("rgbbox"), h, w, spp, j, i, pix[v][j, i], rgb[v][j, i], cam7=cam)
        assert_agrees((frac, bad, f"view {v}: {msg}"), FLOOR_VIEWS[spp])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "random"])
def test_scene_from_arrays_in_scrambled_order(R, name):
    """The caller's spheres in a scrambled order: hits report indices into that order, and frames are unchanged."""
    s, c = scene_arrays(name)
    order = np.random.default_rng(9).permutation(len(s))
    s2 = np.ascontiguousarray(s[order])
    ref = F.Reference(s2, R.host_lbvh(s2), c)
    rays = query_rays(name)
    h, w = 48, 64
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s2, c))
        out = ctx.trace_hits(pr, _dev(rays), t_min=0.0, t_max=1e9)
        got = _np(_torch().cat([out["t"][:, None], out["sphere"].view(_torch().float32)[:, None], out["p"],
                                out["normal"]], 1))
        pix, rgb = ctx.render_host(h, w, pr, 1, want_rgb=True)
    assert_agrees(judge_hits(ref, rays, 0.0, 1e9, got), FLOOR_RAYS[name])
    j, i = pick_pixels(h, w, 800, 5)
    assert_agrees(judge_pixels(ref, h, w, 1, j, i, pix[j, i], rgb[j, i]), FLOOR_SCRAMBLED[name])


def _gpu_sources(ctx, pr):
    torch = _torch()

    def rec(out):
        return _np(torch.cat([out["t"][..., None], out["sphere"].view(torch.float32)[..., None], out["p"], out["normal"]], -1))

    def multi(out):
        return rec(out), _np(out["count"])

    return dict(hits=lambda rays: (lambda lo, hi: rec(ctx.trace_hits(pr, _dev(rays), t_min=lo, t_max=hi))),
                occluded=lambda rays: (lambda lo, hi: _np(ctx.trace_occluded(pr, _dev(rays), t_min=lo, t_max=hi))),
                multi=lambda rays: (lambda lo, hi: multi(ctx.trace_multi_hits(pr, _dev(rays), K, t_min=lo, t_max=hi))),
                ranged_hits=lambda rays: (lambda r8: rec(ctx.trace_hits(pr, _dev(r8)))),
                ranged_occluded=lambda rays: (lambda r8: _np(ctx.trace_occluded(pr, _dev(r8)))),
                ranged_multi=lambda rays: (lambda r8: multi(ctx.trace_multi_hits(pr, _dev(r8), K))))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox", "irreg", "random", "comb"])
def test_ray_queries(R, name):
    rays = comb_rays() if name == "comb" else query_rays(name)
    with R.Context(device=0) as ctx:
        pr = _gpu_prepared(ctx, name, 48, 64)
        src = _gpu_sources(ctx, pr)
        check_queries(reference(name), rays, FLOOR_RAYS[name], *(src[k](rays) for k in
                                               ("hits", "occluded", "multi", "ranged_hits", "ranged_occluded", "ranged_multi")))


@pytest.mark.gpu
@pytest.mark.parametrize("max_depth", [1, 3, 50])
@pytest.mark.parametrize("name", ["rgbbox", "irreg", "random"])
def test_trace_paths(R, name, max_depth):
    rays = query_rays(name)[:1200]
    with R.Context(device=0) as ctx:
        pr = _gpu_prepared(ctx, name, 48, 64)
        rgb, seg = ctx.trace_paths(pr, _dev(rays), max_depth=max_depth)
        rgb, seg = _np(rgb), _np(seg)
    assert_agrees(judge_paths(reference(name), rays, max_depth, rgb, seg), FLOOR_PATHS[name])


@pytest.mark.gpu
def test_comb_frame(R):
    """The comb tree's camera frame: stale boxes on most levels of a 30-level comb over coincident spheres."""
    h, w = 48, 64
    with R.Context(device=0) as ctx:
        pr = _gpu_prepared(ctx, "comb", h, w)
        pix, rgb = ctx.render_host(h, w, pr, 3, want_rgb=True)
    j, i = pick_pixels(h, w, h * w, 0)
    assert_agrees(judge_pixels(reference("comb"), h, w, 3, j, i, pix[j, i], rgb[j, i]), FLOOR_FRAMES["comb", 3])


@pytest.mark.gpu
def test_million_spheres(R):
    """2^20 random spheres on a few hundred camera and random rays.  Most rays pass within a near-tie of some small
    sphere here, so only about a quarter are judged, and paths (a near-tie on any segment) hardly ever are."""
    n = 1 << 20
    s, c = R.host_scene("random", n, 1)
    ref = F.Reference(s, R.host_lbvh(s), c)
    cam = R.camera_rays(R.host_camera(c, 64, 64), 64, 64).reshape(-1, 6)[::17][:200]
    rays = np.ascontiguousarray(np.concatenate([cam, random_rays(s, 100, 3)]), np.float32)
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(64, 64, ctx.scene_random(n, 1))
        src = _gpu_sources(ctx, pr)
        assert_agrees(judge_hits(ref, rays, 0.0, 1e9, src["hits"](rays)(0.0, 1e9)), FLOOR_RAYS["random1M"])
        assert_agrees(judge_occluded(ref, rays, 0.1, 1e9, src["occluded"](rays)(0.1, 1e9)), FLOOR_RAYS["random1M"])
