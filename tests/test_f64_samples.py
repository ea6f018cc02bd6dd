"""Multi-sample outputs against tests/f64_reference.py one sample at a time.

A pixel of an spp-sample frame is judged by f64_reference.Reference.pixels only when every one of its samples is, which
at spp 16 leaves a few per cent of rgbbox's pixels: frames at spp > 1, progressive chunks, adaptive and noise-driven
rendering are almost unjudged that way.  Here each sample is judged on its own instead.  Sample s of every pixel is
taken from the GPU twice, as a one-sample progressive chunk [s, s + 1) on a running sum of +0.0 (the sum is then
+0 + colour_s, from the host's offset table) and as a one-sample adaptive call at count s (from the kernel's own
offsets), for s in [0, 16) and at every window of test_sample_indices.WINDOWS, up to INT32_MAX, without tracing the
samples before a window.  The multi-sample outputs are then tied to those samples bit for bit: frames at spp 3 and 16
and the progressive chain [0, 16) are the in-order f32 fold of the per-sample colours, so every judged sample of theirs
is judged.  M2 of render_adaptive_var is held to the f64 variance of the f64 colours within a stated bound, and
adaptive_select's mask to the f64 statistic wherever that is farther than the bound from the threshold.  The G-buffer
is judged against Reference.gbuffer, and scene batches, frames and ray queries, member by member against each member's
own Reference.

Every case checks its premises first: the plan each call ran, and the judged fraction of its own case against a floor
measured on the oracle's output (CPU) and rounded down.  The CPU cases run the same comparisons on the oracle, and the
mutants of f64_reference that concern these outputs are each rejected there (test_f64_reference runs every mutant)."""
import functools

import numpy as np
import pytest

import f64_reference as F
import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from ray_query_cases import _dev, _np, _torch, bits_differ, random_rays
from test_f64_reference import (K, _oracle_sources, assert_agrees, check_queries, judge_pixels, pick_pixels, reference,
                                scene_arrays, surface_rays, topology)
from test_render_accumulate import frame_of, sequential_sum
from test_render_adaptive_var import m2_model, select_model
from test_render_gbuffer import oracle_gbuffer
from test_sample_indices import WINDOWS, offsets_rule, rays_rule

SAMPLE_SCENES = ["rgbbox", "irreg", "random", "rgbbox_x255"]
SAMPLE_SHAPES = [(37, 53), (48, 160)]
FIRST = np.arange(16)                                                        # s in [0, 16)
WINDOW_INDICES = np.concatenate([start + np.arange(k) for start, k in WINDOWS.values()])
INDICES = np.concatenate([FIRST, WINDOW_INDICES])
SAMPLE_PIXELS = 60           # pixels judged per case (every one of their samples)
VAR_SCENES = ["random", "irreg", "rgbbox_top_down"]
VAR_NS = [8, 16]
# adaptive_select's rules: thresholds of 0.2 % to 1 % relative noise, among irreg's edge pixels (random's pixels are all
# near 0.03 %, within the bound of the threshold)
RULES = [(0.002, 0.0, 2, 1 << 20), (0.005, 0.0, 2, 1 << 20), (0.01, 0.1, 2, 1 << 20)]
GB_CASES = [("rgbbox", None), ("irreg", None), ("random", None), ("rgbbox", "custom")]
GB_CAM = np.float32([25, 5, 28, 0, 0, -20, 40])
BATCH_SHAPE = (40, 72)

# Floors of the judged fractions, measured on the oracle's output (CPU) and rounded down; the lowest over the shapes.
FLOOR_SAMPLES = {"rgbbox": 0.5, "irreg": 0.9, "random": 0.9, "rgbbox_x255": 0.45}         # per sample, s in [0, 16)
FLOOR_WINDOWS = {"rgbbox": 0.45, "irreg": 0.85, "random": 0.95, "rgbbox_x255": 0.45}       # per sample, every window
FLOOR_M2 = {"random": 0.6, "irreg": 0.65, "rgbbox_top_down": 0.95}                         # pixels, all samples judged
FLOOR_SELECT = {"random": 0.6, "irreg": 0.65, "rgbbox_top_down": 0.95}                     # pixels, lowest over RULES
FLOOR_GBUFFER = {1: 0.95, 3: 0.8, 8: 0.65}                                                 # pixels, lowest over GB_CASES
FLOOR_BATCH = {("random", 1): 0.85, ("random", 3): 0.8, ("rgbbox", 1): 0.4, ("rgbbox", 3): 0.15}   # frames, per member
FLOOR_BATCH_RAYS = {"random": 0.95, "rgbbox": 0.95}                                        # every query kind, per member


# ------------------------------------------------------------------------------------------ comparisons


def judge_samples(ref, h, w, j, i, s, got, cam7=None):
    """(judged fraction, disagreements on judged samples, message) of per-sample colours got [len(j), len(s), 3] of
    pixels (j, i) of an h x w frame at sample indices s against the f64 reference."""
    want, err, judged = ref.samples(h, w, np.asarray(j)[:, None], np.asarray(i)[:, None], np.asarray(s)[None, :], cam7)
    got = np.asarray(got, np.float64)
    with np.errstate(invalid="ignore"):
        far = np.abs(got - want) > (4 * err + 1e-6)[..., None] * np.maximum(1.0, np.abs(want))
    bad = judged & (far | (np.isnan(got) != np.isnan(want))).any(-1)
    frac = float(judged.mean())
    k = np.argwhere(bad)[:3]
    msg = (f"judged {frac:.3f} of {judged.size} samples, {int(bad.sum())} judged samples differ"
           + "".join(f"; ({j[p]}, {i[p]}) sample {s[q]} got {got[p, q]} want {want[p, q]}" for p, q in k))
    return frac, int(bad.sum()), msg


def colour_delta(want, err):
    """How far a judged sample's f32 colour may be from its f64 colour: judge_samples' tolerance."""
    return (4 * err + 1e-6)[..., None] * np.maximum(1.0, np.abs(want))


def judge_m2(ref, want, err, judged, S, M2):
    """(judged fraction, disagreements, message) of the sums S [p, 3] and M2 [p, 3] of n samples of p pixels against
    the f64 reference's colours want [p, n, 3] (err, judged [p, n] from Reference.samples): on pixels whose samples are
    all judged, M2 / (n - 1) is the f64 unbiased variance within m2_bound / (n - 1), NaN where it is NaN."""
    n = want.shape[1]
    ok = judged.all(1)
    S_ref, M_ref = ref.m2(want)
    bound = F.m2_bound(want, colour_delta(want, err))
    with np.errstate(invalid="ignore"):
        far = np.abs(M2.astype(np.float64) - M_ref) / (n - 1) > bound / (n - 1)
        far |= np.abs(S.astype(np.float64) - S_ref) > colour_delta(want, err).sum(1) + n * n * F.U32 * np.abs(want).sum(1)
    bad = ok & (far | (np.isnan(M2) != np.isnan(M_ref))).any(-1)
    return float(ok.mean()), int(bad.sum()), f"M2 of {n} samples: judged {ok.mean():.3f} of {len(ok)} pixels, {int(bad.sum())} differ"


def judge_select(ref, want, err, judged, S, M2, n, rule, mask):
    """(judged fraction, disagreements, message) of adaptive_select's mask [p] on sums and M2 of n samples against
    Reference.select on the f64 colours: judged where every sample is and the f64 statistic E is farther from the
    threshold T than E's and T's bounds (m2_bound over n (n - 1); the sums' error through T), or where either is NaN
    (NaN is not above T on both sides).  Also returns the number of judged pixels the f64 rule selects."""
    r, f = rule[0], rule[1]
    S_ref, M_ref = ref.m2(want)
    mask_ref, E, T = ref.select(S_ref, M_ref, np.full(len(S), n), *rule)
    d = colour_delta(want, err)
    bE = F.m2_bound(want, d).sum(-1) / (n * (n - 1)) + 8 * F.U32 * np.abs(E)
    dm = (d.sum(1) + n * n * F.U32 * np.abs(want).sum(1)).sum(-1) / n
    m = np.abs(S_ref.sum(-1) / n + f)
    bT = 2 * r * r * m * dm + r * r * dm * dm + 8 * F.U32 * T
    with np.errstate(invalid="ignore"):
        ok = judged.all(1) & ((np.abs(E - T) > bE + bT) | np.isnan(E) | np.isnan(T))
    bad = ok & (np.asarray(mask, bool) != mask_ref)
    return (float(ok.mean()), int(bad.sum()), f"select {rule}: judged {ok.mean():.3f} of {len(ok)} pixels, "
            f"{int(bad.sum())} differ"), int((ok & mask_ref).sum())


def gbuffer_bad(want, rec, got):
    """Per pixel: the got buffers (numpy dict of [p] / [p, 3]) are not the f64 ones: another id or coverage, or depth,
    normal or albedo further than f32 arithmetic explains (records_bad's tolerances for t and the normal, averaged over
    the samples for the normal)."""
    O, D = rec["O"], rec["D"]
    dn = np.sqrt(F._dot(D, D))
    on = np.sqrt(F._dot(O, O))
    t = np.abs(rec["t"])
    graze = 1e-6 * t / np.sqrt(np.maximum(rec["dm"], 1e-30))
    tol_t = 1e-5 * (t + on / dn + 1.0) + graze
    tol_p = 1e-5 * (t * dn + on + 1.0) + graze * dn
    tol_n = tol_p / np.maximum(np.abs(rec["rad"]), 1e-30) + 1e-5
    with np.errstate(invalid="ignore"):
        bad = (np.asarray(got["id"]) != want["id"]) | (np.asarray(got["coverage"]) != want["coverage"])
        bad |= np.abs(got["depth"] - want["depth"]) > tol_t[:, 0]
        bad |= (np.abs(got["normal"] - want["normal"]) > tol_n.mean(1)[:, None]).any(1)
        bad |= (np.abs(got["albedo"] - want["albedo"]) > 1e-5 * np.maximum(1.0, np.abs(want["albedo"]))).any(1)
    return bad


def judge_gbuffer(ref, h, w, spp, j, i, got, cam7=None):
    want, judged, rec = ref.gbuffer(h, w, j, i, spp, cam7)
    rec["rad"] = ref.rad[np.maximum(rec["leaf"], 0)]
    bad = judged & gbuffer_bad(want, rec, {k: np.asarray(v)[j, i] for k, v in got.items()})
    return (float(judged.mean()), int(bad.sum()),
            f"G-buffer at spp {spp}: judged {judged.mean():.3f} of {len(j)} pixels, {int(bad.sum())} judged pixels differ")


# ------------------------------------------------------------------------------------------ the oracle's samples


@functools.lru_cache(maxsize=None)
def oracle_prepared(name, h, w):
    s, c = scene_arrays(name)
    return Q.prepare_custom(s, c, h, w)


def case_pixels(h, w, name):
    return pick_pixels(h, w, SAMPLE_PIXELS, h * w + len(name))


@functools.lru_cache(maxsize=None)
def oracle_samples(name, h, w, idx):
    """The oracle's path colours of samples idx (a tuple) of the case's pixels: float32 [p, len(idx), 3]."""
    o = oracle_prepared(name, h, w)
    j, i = case_pixels(h, w, name)
    rays = rays_rule(o.camera(), h, w, j[:, None], i[:, None], np.asarray(idx)[None, :])
    return o.trace_paths(rays.reshape(-1, 6))[0].reshape(len(j), len(idx), 3)


# ------------------------------------------------------------------------------------------ CPU: offsets


def test_offsets_follow_the_header_rule(R):
    """F.sample_offsets is the header's f32 rule: the host table bit for bit below 2^16, offsets_rule at every window,
    and apart from the old f64 product there by at least a tenth."""
    s = np.arange(1 << 16)
    ox, oy = F.sample_offsets(s)
    table = R.host_sample_offsets(1 << 16)
    for got, want in ((ox, table[:, 0]), (oy, table[:, 1])):
        assert (got.astype(np.float32).astype(np.float64) == got).all(), "the offsets are f32 values"
        assert bits_differ(got.astype(np.float32), want) == 0
    rx, ry = offsets_rule(WINDOW_INDICES)
    fx, fy = F.sample_offsets(WINDOW_INDICES)
    assert bits_differ(fx.astype(np.float32), rx) == 0 and bits_differ(fy.astype(np.float32), ry) == 0
    mx, my = F.sample_offsets(WINDOW_INDICES, "offsets_in_f64")
    for start, k in WINDOWS.values():
        w = np.isin(WINDOW_INDICES, start + np.arange(k))
        assert max(np.abs(mx - fx)[w].max(), np.abs(my - fy)[w].max()) >= 0.1, start


# ------------------------------------------------------------------------------------------ CPU: the oracle against it


@pytest.mark.parametrize("h,w", SAMPLE_SHAPES)
@pytest.mark.parametrize("name", SAMPLE_SCENES)
def test_oracle_samples(name, h, w):
    j, i = case_pixels(h, w, name)
    for idx, floor in ((FIRST, FLOOR_SAMPLES), (WINDOW_INDICES, FLOOR_WINDOWS)):
        got = oracle_samples(name, h, w, tuple(idx))
        assert_agrees(judge_samples(reference(name), h, w, j, i, idx, got), floor[name])


def _oracle_var(name, n, ref=None):
    """(want, err, judged, S, M2) of the first n samples of the case's pixels: the f64 reference's samples and the M2
    rule on the oracle's colours."""
    h, w = SAMPLE_SHAPES[0]
    j, i = case_pixels(h, w, name)
    ref = reference(name) if ref is None else ref
    want, err, judged = ref.samples(h, w, j[:, None], i[:, None], FIRST[None, :n])
    x = oracle_samples(name, h, w, tuple(FIRST[:n]))
    S, M2, _ = m2_model(x[:, None], [None], [n])
    return want, err, judged, S[:, 0], M2[:, 0]


@pytest.mark.parametrize("n", VAR_NS)
@pytest.mark.parametrize("name", VAR_SCENES)
def test_oracle_m2_and_selection(name, n):
    """M2 and the selection rule over the oracle's colours (m2_model, select_model) against the f64 reference."""
    want, err, judged, S, M2 = _oracle_var(name, n)
    assert_agrees(judge_m2(reference(name), want, err, judged, S, M2), FLOOR_M2[name])
    for rule in RULES:
        mask, _ = select_model(S, M2, np.full(len(S), n, np.int32), *rule)
        result, _ = judge_select(reference(name), want, err, judged, S, M2, n, rule, mask)
        assert_agrees(result, FLOOR_SELECT[name])


def gbuffer_pixels(h, w, spp):
    return pick_pixels(h, w, 300, spp)


def _gb_case(name, camera):
    s, c = scene_arrays(name)
    return s, (GB_CAM if camera == "custom" else c)


@pytest.mark.parametrize("spp", [1, 3, 8])
@pytest.mark.parametrize("name,camera", GB_CASES)
def test_oracle_gbuffer(name, camera, spp):
    """test_render_gbuffer's rule over the CPU oracle against Reference.gbuffer."""
    h, w = 37, 53
    s, c = _gb_case(name, camera)
    got = oracle_gbuffer(Q.prepare_custom(s, c, h, w), s[:, 3:6], h, w, spp)
    j, i = gbuffer_pixels(h, w, spp)
    assert_agrees(judge_gbuffer(reference(name), h, w, spp, j, i, got, c), FLOOR_GBUFFER[spp])


# ------------------------------------------------------------------------------------------ CPU: scene batch members


def batch_members(kind):
    """(spheres float32 [3, n, 7], cameras float32 [3, 7], references) of a scene batch: random(3000) of three seeds, or
    rgbbox seen from three cameras."""
    import raytracers_b200 as R
    if kind == "random":
        scenes = [R.host_scene("random", 3000, seed) for seed in (1, 2, 3)]
        refs = [F.Reference(s, R.host_lbvh(s), c) for s, c in scenes]
    else:
        s, c = scene_arrays("rgbbox")
        scenes = [(s, c), (s, np.float32([-20, 20, 10, 5, -10, -25, 100])), (s, GB_CAM)]
        refs = [F.Reference(s, topology("rgbbox"), cam) for _, cam in scenes]
    return (np.ascontiguousarray(np.stack([s for s, _ in scenes]), np.float32),
            np.ascontiguousarray(np.stack([c for _, c in scenes]), np.float32), refs)


@functools.lru_cache(maxsize=None)
def _batch(kind):
    return batch_members(kind)


@functools.lru_cache(maxsize=None)
def batch_rays(kind, b):
    """Rays of member b: random rays, the member's camera rays and rays from just outside its spheres: float32 [700, 6]."""
    import raytracers_b200 as R
    s, cams, _ = _batch(kind)
    h, w = BATCH_SHAPE
    cam = R.camera_rays(R.host_camera(cams[b], h, w), h, w).reshape(-1, 6)
    cam = cam[np.random.default_rng(20 + b).choice(len(cam), 300, replace=False)]
    return np.ascontiguousarray(np.concatenate([random_rays(s[b], 250, 21 + b), cam, surface_rays(s[b], 150, 22 + b)]),
                                np.float32)


BATCH_QUERIES = ("hits", "occluded", "multi", "ranged_hits", "ranged_occluded", "ranged_multi")


@pytest.mark.parametrize("kind", ["random", "rgbbox"])
def test_oracle_scene_batch_members(kind):
    """Each member's frames at spp 1 and 3 and its ray queries on the oracle, against the member's own reference."""
    from oracle import pyoracle as O
    s, cams, refs = _batch(kind)
    h, w = BATCH_SHAPE
    j, i = pick_pixels(h, w, 200, 8)
    for b, ref in enumerate(refs):
        for spp in (1, 3):
            pix, rgb, _ = O.Scene.custom(s[b], cams[b]).prepare(h, w).render(h, w, spp=spp, want_rgb=True)
            frac, bad, msg = judge_pixels(ref, h, w, spp, j, i, pix[j, i], rgb[j, i])
            assert_agrees((frac, bad, f"member {b}: {msg}"), FLOOR_BATCH[kind, spp])
        rays = batch_rays(kind, b)
        src = _oracle_sources(Q.prepare_custom(s[b], cams[b], h, w))
        check_queries(ref, rays, FLOOR_BATCH_RAYS[kind], *(src[k](rays) for k in BATCH_QUERIES))


# ------------------------------------------------------------------------------------------ CPU: mutants


def _mutant_window(mutant):
    """The oracle's samples of irreg's 2^21/cx window against the reference with f64 offsets."""
    start, k = WINDOWS["2^21/cx"]
    idx = start + np.arange(k)
    h, w = SAMPLE_SHAPES[0]
    j, i = case_pixels(h, w, "irreg")
    return judge_samples(reference("irreg", mutant), h, w, j, i, idx, oracle_samples("irreg", h, w, tuple(idx)))


def _mutant_m2(mutant):
    want, err, judged, S, M2 = _oracle_var("irreg", 16, reference("irreg", mutant))
    return judge_m2(reference("irreg", mutant), want, err, judged, S, M2)


def _mutant_select(mutant):
    want, err, judged, S, M2 = _oracle_var("irreg", 16)
    ref = reference("irreg", mutant)
    results = []
    for rule in RULES:
        mask, _ = select_model(S, M2, np.full(len(S), 16, np.int32), *rule)
        results.append(judge_select(ref, want, err, judged, S, M2, 16, rule, mask)[0])
    return min(r[0] for r in results), sum(r[1] for r in results), "; ".join(r[2] for r in results)


def _mutant_gbuffer(mutant):
    h, w, spp = 37, 53, 3
    s, c = scene_arrays("irreg")
    got = oracle_gbuffer(oracle_prepared("irreg", h, w), s[:, 3:6], h, w, spp)
    j, i = gbuffer_pixels(h, w, spp)
    return judge_gbuffer(reference("irreg", mutant), h, w, spp, j, i, got)


MUTANT_CASES = {
    "offsets_in_f64": _mutant_window,
    "welford_old_mean": _mutant_m2,
    "select_without_count": _mutant_select,
    "gbuffer_depth_last_sample": _mutant_gbuffer,
    "gbuffer_id_in_leaf_order": _mutant_gbuffer,
    "gbuffer_miss_albedo_black": _mutant_gbuffer,
}


# ------------------------------------------------------------------------------------------ GPU: per-sample colours


def _prepared(ctx, name, h, w, cam=None):
    s, c = scene_arrays(name)
    return ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c if cam is None else cam))


def gpu_samples(ctx, pr, h, w, idx):
    """Sample s of every pixel for each s of idx, as a progressive chunk [s, s + 1) on a sum of +0.0 and as an adaptive
    call of one sample at count s on a sum of +0.0: numpy float32 [h, w, len(idx), 3] each, and the calls' plans."""
    torch = _torch()
    k = len(idx)
    acc = torch.zeros((k, h, w, 3), dtype=torch.float32, device="cuda")
    ada = torch.zeros((k, h, w, 3), dtype=torch.float32, device="cuda")
    cnt = torch.from_numpy(np.repeat(np.asarray(idx, np.int32), h * w).reshape(k, h, w)).cuda()
    torch.cuda.synchronize()
    plans = []
    for q, s in enumerate(idx):
        ctx.render_accumulate_into(acc[q].data_ptr(), h, w, pr, int(s), int(s) + 1)
        plans.append(ctx.last_plan())
        ctx.render_adaptive_into(ada[q].data_ptr(), cnt[q].data_ptr(), h, w, pr, 1)
        plans.append(ctx.last_plan())
    ctx.sync()
    assert (_np(cnt) == np.asarray(idx)[:, None, None] + 1).all(), "every adaptive call added one sample"
    return _np(acc.permute(1, 2, 0, 3)), _np(ada.permute(1, 2, 0, 3)), plans


def _frame(ctx, pr, h, w, spp):
    torch = _torch()
    pix = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    rgb = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.render_into(pix.data_ptr(), h, w, pr, spp, rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb), ctx.last_plan()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SAMPLE_SHAPES)
@pytest.mark.parametrize("name", SAMPLE_SCENES)
def test_samples_and_the_frames_they_make(R, name, h, w):
    """Per-sample colours of s in [0, 16) and every window, from chunks and adaptive calls, judged; then frames at
    spp 3 and 16 and the progressive chain [0, 16), spread (the default) and pixel-bound (wq_spread 0), equal to the
    in-order f32 fold of the per-sample colours, the sum bit for bit and then the quantised pixel."""
    torch = _torch()
    j, i = case_pixels(h, w, name)
    first = None
    for spread in (1, 0):
        with R.Context(device=0, wq_spread=spread) as ctx:
            pr = _prepared(ctx, name, h, w)
            acc, ada, plans = gpu_samples(ctx, pr, h, w, INDICES)
            assert [(p["query"], p["spread"]) for p in plans] == [("accumulate", 0), ("adaptive", 0)] * len(INDICES), \
                "one sample per pixel is pixel-bound"
            assert bits_differ(acc, ada) == 0, f"spread {spread}: the host table and the in-kernel offsets differ"
            if first is None:
                for idx, floor, sl in ((FIRST, FLOOR_SAMPLES, slice(0, 16)), (WINDOW_INDICES, FLOOR_WINDOWS, slice(16, None))):
                    assert_agrees(judge_samples(reference(name), h, w, j, i, idx, acc[j, i][:, sl]), floor[name])
                first = acc
            else:
                assert bits_differ(acc, first) == 0, "the samples do not depend on the context's plan options"
            colours = acc[:, :, :16]
            for spp in (3, 16):
                pix, rgb, p = _frame(ctx, pr, h, w, spp)
                assert (p["query"], p["spread"]) == ("pixels", spread), p
                want_pix, want_rgb = frame_of(sequential_sum(colours, 0, spp), spp)
                assert bits_differ(rgb, want_rgb) == 0 and (pix == want_pix).all(), f"spread {spread}: frame at spp {spp}"
            accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
            for a, b in ((0, 1), (1, 3), (3, 16)):
                pix, rgb = ctx.render_accumulate(pr, accum, a, b, want_rgb=True)
                p = ctx.last_plan()
                assert (p["query"], p["spread"]) == ("accumulate", int(spread and b - a > 1)), p
            want = sequential_sum(colours, 0, 16)
            assert bits_differ(_np(accum), want) == 0, f"spread {spread}: the chain's sums"
            want_pix, want_rgb = frame_of(want, 16)
            assert bits_differ(_np(rgb), want_rgb) == 0 and (_np(pix) == want_pix).all(), f"spread {spread}: the chain's frame"


# ------------------------------------------------------------------------------------------ GPU: M2 and selection


@pytest.mark.gpu
@pytest.mark.parametrize("n", VAR_NS)
@pytest.mark.parametrize("name", VAR_SCENES)
def test_m2_and_selection(R, name, n):
    """render_adaptive_var over n samples in one spread call, M2 and the sums against the f64 colours, and
    adaptive_select's mask against the f64 statistic, on the pixels and within the bounds of judge_m2 / judge_select."""
    torch = _torch()
    h, w = SAMPLE_SHAPES[0]
    j, i = case_pixels(h, w, name)
    ref = reference(name)
    want, err, judged = ref.samples(h, w, j[:, None], i[:, None], FIRST[None, :n])
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, name, h, w)
        accum = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
        m2 = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        ctx.render_adaptive(pr, accum, counts, n, m2=m2)
        p = ctx.last_plan()
        assert (p["query"], p["spread"]) == ("adaptive_var", 1), p
        assert (_np(counts) == n).all()
        S, M2 = _np(accum)[j, i], _np(m2)[j, i]
        assert_agrees(judge_m2(ref, want, err, judged, S, M2), FLOOR_M2[name])
        decided = 0
        for rule in RULES:
            mask, n_sel = ctx.adaptive_select(accum, m2, counts, *rule)
            result, selected = judge_select(ref, want, err, judged, S, M2, n, rule, _np(mask)[j, i])
            assert_agrees(result, FLOOR_SELECT[name])
            decided += selected
        if name == "irreg":   # random's noise is all within the bound of these thresholds, rgbbox_top_down's is NaN
            assert decided > 0, "some judged pixel is selected by some rule"


# ------------------------------------------------------------------------------------------ GPU: G-buffer


@pytest.mark.gpu
@pytest.mark.parametrize("name,camera", GB_CASES)
def test_gbuffer(R, name, camera):
    h, w = 37, 53
    s, c = _gb_case(name, camera)
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        for spp in (1, 3, 8):
            got = {k: _np(v) for k, v in ctx.render_gbuffer(pr, h, w, spp).items()}
            assert ctx.last_plan()["query"] == "gbuffer"
            j, i = gbuffer_pixels(h, w, spp)
            frac, bad, msg = judge_gbuffer(reference(name), h, w, spp, j, i, got, c)
            assert_agrees((frac, bad, f"{name} {camera or ''}: {msg}"), FLOOR_GBUFFER[spp])


# ------------------------------------------------------------------------------------------ GPU: scene batches


def _batch_sources(ctx, batch, b, B):
    """Query sources (as _gpu_sources) of member b: the batch query of every member's rays, member b's answers."""
    torch = _torch()

    def stack(rays):   # every member traces the same rays
        return _dev(np.stack([rays] * B))

    def rec(out):
        return _np(torch.cat([out["t"][..., None], out["sphere"].view(torch.float32)[..., None], out["p"],
                              out["normal"]], -1)[b])

    def multi(out):
        return rec(out), _np(out["count"][b])

    return dict(hits=lambda rays: (lambda lo, hi: rec(ctx.trace_scene_batch_hits(batch, stack(rays), lo, hi))),
                occluded=lambda rays: (lambda lo, hi: _np(ctx.trace_scene_batch_occluded(batch, stack(rays), lo, hi)[b])),
                multi=lambda rays: (lambda lo, hi: multi(ctx.trace_scene_batch_multi_hits(batch, stack(rays), K, lo, hi))),
                ranged_hits=lambda rays: (lambda r8: rec(ctx.trace_scene_batch_hits(batch, stack(r8)))),
                ranged_occluded=lambda rays: (lambda r8: _np(ctx.trace_scene_batch_occluded(batch, stack(r8))[b])),
                ranged_multi=lambda rays: (lambda r8: multi(ctx.trace_scene_batch_multi_hits(batch, stack(r8), K))))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "rgbbox"])
def test_scene_batch_members(R, kind):
    """Frames at spp 1 and 3 and closest-hit, occlusion and multi-hit queries (per-call and per-ray intervals) of a
    scene batch, each member against its own reference."""
    s, cams, refs = _batch(kind)
    h, w = BATCH_SHAPE
    j, i = pick_pixels(h, w, 200, 8)
    with R.Context(device=0) as ctx:
        batch = ctx.prepare_scene_batch(h, w, _dev(s), cams)
        for spp in (1, 3):
            pix, rgb = ctx.render_scene_batch(batch, h, w, spp, want_rgb=True)
            assert ctx.last_plan()["query"] == "scene_batch"
            pix, rgb = _np(pix), _np(rgb)
            for b, ref in enumerate(refs):
                frac, bad, msg = judge_pixels(ref, h, w, spp, j, i, pix[b][j, i], rgb[b][j, i])
                assert_agrees((frac, bad, f"member {b}: {msg}"), FLOOR_BATCH[kind, spp])
        for b, ref in enumerate(refs):
            rays = batch_rays(kind, b)
            src = _batch_sources(ctx, batch, b, len(refs))
            check_queries(ref, rays, FLOOR_BATCH_RAYS[kind], *(src[k](rays) for k in BATCH_QUERIES))
        assert ctx.last_plan()["query"] == "scene_batch_multihit"
        batch.free()
