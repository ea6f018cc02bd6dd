"""Adaptive rendering driven by a noise estimate (include/ray_b200.h ray_b200_render_adaptive_var and
ray_b200_adaptive_select).  render_adaptive_var is render_adaptive plus m2, each pixel's per-channel M2 (Welford's running
f32 sum of squared deviations from the mean), updated one sample at a time in sample order whatever the chunking;
adaptive_select turns accum, m2 and counts into the mask of the pixels whose noise estimate is still above the target.

On the CPU the M2 rule is restated in numpy f32 over ragged masked chains of the oracle's per-sample colours, checked to be
Welford's (M2 / (n - 1) is the sample variance), and the selection rule is restated on crafted buffers.  On the GPU
accum, counts and the outputs equal render_adaptive's bit for bit, m2 equals the numpy rule on the GPU's own trace_paths
colours bit for bit (NaN-aware), and the mask and count equal the numpy selection rule."""
import numpy as np
import pytest

import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
from ray_query_cases import PLANS, _dev, _np, _torch, bits_differ
from test_render_accumulate import SCENES, _ctx, _gpu_colours, _one_shot, frame_of
from test_render_adaptive import INT32_MAX, SENTINEL, _adaptive_chain, ragged_model, random_masks
from test_staging_plans import FORCED_PLANS, H, W, _camera_rays, expect, forced, variant  # noqa: F401 (forced: fixture)


def m2_model(colours, masks, n_adds, accum=None, m2=None, counts=None):
    """The M2 rule on the CPU: colours [h, w, S, 3]; per call, every selected pixel with a valid count c gets samples
    [c, c + n) added one at a time, M2 = +0 after sample 0 and M2 += (x_k - S_k / k) * (x_k - S_{k+1} / (k + 1)) after
    sample k >= 1, all in f32.  Returns (accum, m2, counts)."""
    h, w = colours.shape[:2]
    acc = np.zeros((h, w, 3), np.float32) if accum is None else accum.astype(np.float32).copy()
    m2 = np.zeros((h, w, 3), np.float32) if m2 is None else m2.astype(np.float32).copy()
    cnt = np.zeros((h, w), np.int64) if counts is None else counts.astype(np.int64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for mask, n in zip(masks, n_adds):
            sel = np.ones((h, w), bool) if mask is None else mask.astype(bool)
            sel &= (cnt >= 0) & (cnt <= INT32_MAX - n)
            for c in np.unique(cnt[sel]):
                p = sel & (cnt == c)
                a, m, xs = acc[p], m2[p], colours[p]
                for k in range(int(c), int(c) + n):
                    x = xs[:, k, :]
                    if k == 0:
                        a, m = x.copy(), np.zeros_like(x)
                    else:
                        nxt = a + x
                        m = m + (x - a / np.float32(k)) * (x - nxt / np.float32(k + 1))
                        a = nxt
                acc[p], m2[p] = a, m
            cnt[sel] += n
    return acc, m2, cnt.astype(np.int32)


def select_model(accum, m2, counts, rel_err, mean_floor, min_count, max_count):
    """The selection rule of ray_b200_adaptive_select in numpy f32: (mask, number of ones)."""
    n = counts.astype(np.int64)
    S, M = accum.astype(np.float32), m2.astype(np.float32)
    nf, nf1 = n.astype(np.float32), (n - 1).astype(np.float32)
    r, f = np.float32(rel_err), np.float32(mean_floor)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        v = (M[..., 0] + M[..., 1]) + M[..., 2]
        e = v / (nf * nf1)
        m = ((S[..., 0] + S[..., 1]) + S[..., 2]) / nf + f
        t = (r * m) * (r * m)
        sel = (n >= 0) & (n < max_count) & ((n < min_count) | (e > t))
    return sel, int(sel.sum())


def _pixel_rays(R, camera, h, w, js, iss, spp):
    """camera_rays of the pixels (js[k], iss[k]) of an h x w frame only: float32 [len(js)][spp][6]"""
    c = np.asarray(camera, np.float32).reshape(12)
    f = np.float32
    off = R.host_sample_offsets(spp)
    u = (np.asarray(iss, np.float32)[:, None] + off[:, 0][None, :]) / f(w)
    v = ((f(h) - np.asarray(js, np.float32))[:, None] + off[:, 1][None, :]) / f(h)
    out = np.empty((len(js), spp, 6), np.float32)
    out[..., 0:3] = c[0:3]
    for a in range(3):
        out[..., 3 + a] = ((c[3 + a] + u * c[6 + a]) + v * c[9 + a]) - c[a]
    return out


def _scene_colours(R, scene, h, w, spp):
    s, c = SCENES[scene]()
    o = Q.prepare_custom(s, c, h, w)
    return o.trace_paths(R.camera_rays(o.camera(), h, w, spp).reshape(-1, 6))[0].reshape(h, w, spp, 3)


# ------------------------------------------------------------------------------------------ CPU: the arithmetic


@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "rgbbox_negative"])
def test_m2_model_over_ragged_oracle_chains(R, scene):
    """The numpy rule over ragged masked chains: its sums are render_adaptive's model's, its M2 is independent of the
    chunking (the same per-sample update whatever the calls), and M2 / (n - 1) is the float64 sample variance."""
    h, w = 40, 56
    n_adds = [1, 3, 2, 1, 4]
    colours = _scene_colours(R, scene, h, w, sum(n_adds))
    masks = random_masks(h, w, len(n_adds), 5, 0.6)
    masks[1] = None
    acc, m2, cnt = m2_model(colours, masks, n_adds)
    want_acc, want_cnt = ragged_model(colours, masks, n_adds)
    assert len(np.unique(cnt)) >= 4
    assert (cnt == want_cnt).all() and bits_differ(acc, want_acc) == 0
    for n in np.unique(cnt):
        p = cnt == n
        if n == 0:
            continue
        one_call = m2_model(colours[p][None], [None], [int(n)])[1][0]
        assert bits_differ(m2[p], one_call) == 0, f"count {n}: M2 depends on the chunking"
        if n >= 2:
            x = colours[p][:, :n, :].astype(np.float64)
            with np.errstate(invalid="ignore", over="ignore"):
                var = x.var(axis=1, ddof=1)
            got = m2[p].astype(np.float64) / (n - 1)
            fin = np.isfinite(x).all(axis=1) & (np.abs(x).max(axis=1) < 1e15)    # (f32 overflows beyond, as it may)
            assert fin.sum() > 100
            assert np.allclose(got[fin], var[fin], rtol=1e-3, atol=1e-6), f"count {n}: M2 / (n - 1) is not the sample variance"
        else:
            assert (m2[p].view(np.uint32) == 0).all(), "+0 after sample 0"


def test_welford_survives_where_the_sum_of_squares_cancels():
    """512 samples around a mean far from 0: Welford's M2 in f32 keeps the variance, M2/n - mean^2 in f32 does not."""
    rng = np.random.default_rng(1)
    x = (np.float32(0.9) + np.float32(1e-3) * rng.standard_normal((64, 512, 3))).astype(np.float32)
    _, m2, _ = m2_model(x[:, None], [None], [512])
    var = x.astype(np.float64).var(axis=1, ddof=1)
    assert np.allclose(m2[:, 0].astype(np.float64) / 511, var, rtol=1e-2)
    sq = np.zeros((64, 3), np.float32)
    s = np.zeros((64, 3), np.float32)
    for k in range(512):
        s, sq = s + x[:, k], sq + x[:, k] * x[:, k]
    naive = (sq / np.float32(512) - (s / np.float32(512)) ** 2).astype(np.float64) * 512 / 511
    assert not np.allclose(naive, var, rtol=1e-1)


def crafted_buffers(min_count, max_count, seed=0):
    """Counts around the edges of the rule, zero means, +-inf and NaN in accum and m2, and random pixels."""
    rng = np.random.default_rng(seed)
    counts = np.array([-(2 ** 31), -5, -1, 0, 1, min_count - 1, min_count, min_count + 1, max_count - 1, max_count,
                       max_count + 1, INT32_MAX], np.int64)
    counts = np.clip(counts, -(2 ** 31), INT32_MAX)
    special = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-30, 1e30, 0.5, 3.0])
    n_px = 4096
    cnt = np.concatenate([counts, rng.integers(min_count, max_count, n_px - len(counts))])
    pick = rng.random(n_px) < 0.2
    pick[:len(counts)] = False
    cnt[pick] = rng.choice(counts, int(pick.sum()))
    mean = rng.uniform(0, 1, (n_px, 3)).astype(np.float32)
    acc = (mean * np.maximum(cnt, 1)[:, None]).astype(np.float32)
    m2 = (rng.uniform(0, 1e-3, (n_px, 3)) * np.maximum(cnt - 1, 1)[:, None]).astype(np.float32)
    cnt = cnt.astype(np.int32)
    acc[rng.random(n_px) < 0.05] = 0.0                                           # zero means
    for buf in (acc, m2):
        pick = rng.random((n_px, 3)) < 0.05
        buf[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    return acc.reshape(64, 64, 3), m2.reshape(64, 64, 3), cnt.reshape(64, 64)


def test_select_model_on_crafted_buffers():
    """The rule's edges as the numpy restatement sees them; the GPU test holds the kernel to the same function."""
    acc, m2, cnt = crafted_buffers(8, 64)
    sel, n = select_model(acc, m2, cnt, 0.02, 0.1, 8, 64)
    c = cnt.ravel()
    s = sel.ravel()
    assert not s[c < 0].any() and not s[c >= 64].any()
    assert s[(c >= 0) & (c < 8)].all(), "below min_count: selected whatever the buffers hold"
    assert n == int(s.sum())
    nan_px = np.isnan(acc).any(-1) | np.isnan(m2).any(-1)
    nan_px &= (cnt >= 8) & (cnt < 64)
    assert not sel[nan_px].any(), "a NaN estimate is not selected"
    # mean_floor 0 with a zero mean and zero variance: E = 0 is not above T = 0; any variance is
    a = np.zeros((1, 2, 3), np.float32)
    m = np.float32([[[0, 0, 0], [0, 1e-30, 0]]])
    assert select_model(a, m, np.int32([[16, 16]]), 0.5, 0.0, 8, 64)[0].tolist() == [[False, True]]


def test_python_argument_checks(R):
    torch = _torch()

    class NoContext:
        device = 0

    h, w = 6, 10
    accum, counts = torch.zeros((h, w, 3)), torch.zeros((h, w), dtype=torch.int32)
    for bad in (accum, np.zeros((h, w, 3), np.float32), None, accum[:, :, :2]):
        with pytest.raises(ValueError):
            R.Context.adaptive_select(NoContext(), bad, accum, counts, 0.1, 0.1, 2, 8)
    if not torch.cuda.is_available():
        return
    a = torch.zeros((h, w, 3), device="cuda")
    m2 = torch.zeros((h, w, 3), device="cuda")
    c = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    bad_m2 = [m2.double(), m2.transpose(0, 1), m2[:, :, :2], m2.reshape(h, w * 3), m2.cpu()]
    for bad in bad_m2:
        with pytest.raises(ValueError):
            R.Context.render_adaptive(NoContext(), None, a, c, 1, m2=bad)
        with pytest.raises(ValueError):
            R.Context.adaptive_select(NoContext(), a, bad, c, 0.1, 0.1, 2, 8)
    bad_select = [dict(accum=a.double()), dict(accum=a[:, :, :2]), dict(counts=c.cpu()), dict(counts=c.long()),
                  dict(counts=c[:, :-1]), dict(out=torch.zeros((h, w), device="cuda")),
                  dict(out=torch.zeros((h, w + 1), dtype=torch.bool, device="cuda")),
                  dict(out=torch.zeros((w, h), dtype=torch.bool, device="cuda").t())]
    for change in bad_select:
        args = dict(dict(accum=a, m2=m2, counts=c, out=None), **change)
        with pytest.raises(ValueError):
            R.Context.adaptive_select(NoContext(), args["accum"], args["m2"], args["counts"], 0.1, 0.1, 2, 8, out=args["out"])


# ------------------------------------------------------------------------------------------ GPU helpers


def _var_chain(ctx, pr, h, w, masks, n_adds, accum=None, m2=None, counts=None, check_untouched=False):
    """render_adaptive(m2=...) once per (mask, n_add) on one set of buffers (NaN-filled sums and M2, zero counts,
    sentinel outputs unless given).  With check_untouched, asserts after every call that the pixels it did not select
    kept all five values.  Returns numpy (accum, m2, counts, pixels, rgb)."""
    torch = _torch()
    nan3 = lambda: torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
    accum = nan3() if accum is None else accum
    m2 = nan3() if m2 is None else m2
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda") if counts is None else counts
    pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    for mask, n in zip(masks, n_adds):
        bufs = (accum, m2, counts, pix, rgb)
        before = [t.clone() for t in bufs] if check_untouched else None
        m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else torch.from_numpy(np.asarray(mask, bool)).cuda())
        ctx.render_adaptive(pr, accum, counts, n, mask=m, pixels=pix, rgb=rgb, m2=m2)
        assert ctx.last_plan()["query"] == "adaptive_var"
        if check_untouched and m is not None:
            off = ~m.bool()
            for t0, t in zip(before, bufs):
                assert torch.equal(t0.view(torch.int32)[off], t.view(torch.int32)[off]), "an unselected pixel changed"
    return _np(accum), _np(m2), _np(counts), _np(pix), _np(rgb)


def _check_chain(R, ctx, pr, h, w, masks, n_adds, what, **kw):
    """The chain through render_adaptive(m2=...) against the same chain through render_adaptive (accum, counts,
    outputs) and against the numpy M2 rule on the GPU's own per-sample colours.  Returns (counts, m2)."""
    acc, m2, cnt, pix, rgb = _var_chain(ctx, pr, h, w, masks, n_adds, **kw)
    a0, c0, p0, r0 = _adaptive_chain(ctx, pr, h, w, masks, n_adds)
    assert (cnt == c0).all(), f"{what}: counts"
    sel = cnt > 0
    assert bits_differ(acc[sel], a0[sel]) == 0 and (pix == p0).all() and bits_differ(rgb, r0) == 0, f"{what}: as render_adaptive"
    colours = _gpu_colours(R, ctx, pr, h, w, int(cnt.max()))
    _, want_m2, _ = m2_model(colours, masks, n_adds)
    assert bits_differ(m2[sel], want_m2[sel]) == 0, f"{what}: m2, {bits_differ(m2[sel], want_m2[sel])} values differ"
    assert np.isnan(m2[~sel]).all(), f"{what}: m2 of a pixel no call selected"
    return cnt, m2


# ------------------------------------------------------------------------------------------ GPU: chains


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "rgbbox_x255"])
def test_ragged_chains(R, scene):
    h, w = 150, 211
    ctx, pr = _ctx(R, scene, h, w)
    masks = random_masks(h, w, 6, 21, 0.4)
    never = np.zeros((h, w), bool)
    never[10:30, 40:90] = True
    for m in masks:
        m &= ~never
    masks[0] = masks[0] | ~never      # most pixels start with one sample, so later calls continue from counts 1 to 13
    cnt, _ = _check_chain(R, ctx, pr, h, w, masks, [1, 2, 5, 1, 3, 2], scene)
    _var_chain(ctx, pr, h, w, masks, [1, 2, 5, 1, 3, 2], check_untouched=True)
    assert (cnt[never] == 0).all() and len(np.unique(cnt)) >= 8
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [1, 0])
def test_both_sample_paths(R, spread):
    """Calls of 1 (pixel-bound), 2 to 64 samples, spread or, with wq_spread 0, pixel-bound."""
    h, w = 37, 53
    ctx, pr = _ctx(R, "irreg", h, w, wq_spread=spread)
    masks = [None] + random_masks(h, w, 4, 2, 0.5)
    _check_chain(R, ctx, pr, h, w, masks, [1, 1, 7, 64, 2], f"wq_spread {spread}")
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_add", [1, 4])
def test_caller_supplied_sums_and_m2(R, n_add):
    """The update is f32 arithmetic on whatever accum and m2 hold at each pixel's count: random floats, +-0, +-inf, NaN."""
    torch = _torch()
    h, w = 37, 53
    ctx, pr = _ctx(R, "rgbbox_negative", h, w)
    rng = np.random.default_rng(n_add)
    start_counts = rng.integers(1, 7, (h, w)).astype(np.int32)
    colours = _gpu_colours(R, ctx, pr, h, w, int(start_counts.max()) + n_add)
    special = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan])
    seeded = []
    for _ in range(2):
        b = rng.standard_normal((h, w, 3)).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, (h, w, 3))
        pick = rng.random((h, w, 3)) < 0.3
        b[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
        seeded.append(b)
    mask = rng.random((h, w)) < 0.7
    want_acc, want_m2, want_cnt = m2_model(colours, [mask], [n_add], seeded[0], seeded[1], start_counts)
    acc, m2, cnt, pix, _ = _var_chain(ctx, pr, h, w, [mask], [n_add], _dev(seeded[0]).reshape(h, w, 3),
                                      _dev(seeded[1]).reshape(h, w, 3), torch.from_numpy(start_counts).cuda())
    assert bits_differ(acc, want_acc) == 0 and (cnt == want_cnt).all()
    assert bits_differ(m2, want_m2) == 0
    assert bits_differ(m2[~mask], seeded[1][~mask]) == 0 and (pix[~mask] == SENTINEL).all()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS + [{"wq_packet": 24}, {"wq_packet": 0}], ids=str)
def test_every_plan(R, plan):
    h, w = 203, 301
    ctx, pr = _ctx(R, "irreg", h, w, **plan)
    _check_chain(R, ctx, pr, h, w, [None] + random_masks(h, w, 2, 11), [1, 4, 11], str(plan))
    ctx.close()


@pytest.mark.gpu
def test_forced_boundaries(R, forced):
    """Every stage_cap point at K = 1 / 2, spread samples or not, with and without the packet walk: a one-sample call on
    half the pixels, then a two-sample call on all of them.  m2 against the numpy rule on the oracle's colours; the plan is
    render_adaptive's but for its query; the launched kAdaptiveVar instantiations are exactly the 24 reachable ones."""
    torch = _torch()
    case, launched = forced["case"], set()
    colours = case.oracle.trace_paths(_camera_rays(R, case.oracle.camera(), 3))[0].reshape(H, W, 3, 3)
    half_np = random_masks(H, W, 1, 3)[0]
    half = torch.from_numpy(half_np).cuda()
    want_acc, want_m2, want_cnt = m2_model(colours, [half_np, None], [1, 2])
    for cap_name, cap, nodes, spheres in forced["caps"]:
        for plan in FORCED_PLANS:
            for packet in (0, 8):
                for spread in (1, 0):
                    what = f"{cap_name} (stage_cap {cap}), {plan}, wq_packet {packet}, wq_spread {spread}"
                    with R.Context(device=0, stage_cap=cap, wq_packet=packet, wq_spread=spread, **plan) as ctx:
                        pr = case.prepare(ctx)
                        nan3 = lambda: torch.full((H, W, 3), float("nan"), dtype=torch.float32, device="cuda")
                        accum, m2 = nan3(), nan3()
                        counts = torch.zeros((H, W), dtype=torch.int32, device="cuda")
                        a0 = nan3()
                        c0 = torch.zeros((H, W), dtype=torch.int32, device="cuda")
                        for mask, n in ((half, 1), (None, 2)):
                            ctx.render_adaptive(pr, a0, c0, n, mask=mask)
                            p0 = dict(ctx.last_plan())
                            ctx.render_adaptive(pr, accum, counts, n, mask=mask, m2=m2)
                            p = ctx.last_plan()
                            expect(p, f"{what}, n_add {n}", query="adaptive_var", spread=int(spread and n > 1),
                                   smem_nodes=nodes, smem_spheres=spheres, packet=packet)
                            assert {k: v for k, v in p.items() if k != "query"} == {k: v for k, v in p0.items() if k != "query"}, what
                            launched.add(variant(p))
                        assert (_np(counts) == want_cnt).all(), what
                        assert bits_differ(_np(accum), want_acc) == 0, f"{what}: sums"
                        assert bits_differ(_np(m2), want_m2) == 0, f"{what}: m2"
    reachable = {("adaptive_var", False, k, sp, pk, st) for k in (1, 2) for sp in (False, True) for pk in (False, True)
                 for st in ("partial", "nodes", "whole")}
    assert launched == reachable and len(reachable) == 24, sorted(reachable ^ launched)


# ------------------------------------------------------------------------------------------ GPU: the selection pass


def _select_gpu(ctx, acc, m2, cnt, *rule):
    torch = _torch()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    mask, n = ctx.adaptive_select(t(acc), t(m2), t(cnt), *rule)
    return _np(mask), int(n.item())


@pytest.mark.gpu
def test_select_equals_the_rule(R):
    """Random and crafted buffers, several rules: mask and count bit for bit; one launch; plan and timing unchanged."""
    torch = _torch()
    ctx, pr = _ctx(R, "irreg", 37, 53)
    out = torch.empty((37, 53), dtype=torch.int32, device="cuda")
    ctx.render_into(out.data_ptr(), 37, 53, pr, spp=2)
    ctx.sync()
    plan, ms = ctx.last_plan(), ctx.last_render_ms()
    rng = np.random.default_rng(4)
    bufs = [crafted_buffers(8, 64, seed) for seed in range(3)]
    h, w = 301, 203
    cnt = rng.integers(-3, 80, (h, w)).astype(np.int32)
    acc = (rng.uniform(0, 1, (h, w, 3)) * np.maximum(cnt, 1)[..., None]).astype(np.float32)
    m2 = (rng.exponential(1e-2, (h, w, 3)) * np.maximum(cnt - 1, 1)[..., None]).astype(np.float32)
    bufs.append((acc, m2, cnt))
    rules = [(0.02, 0.1, 8, 64), (0.01, 0.0, 2, 3), (0.5, 0.0, 8, 64), (0.0, 0.0, 16, 80), (0.1, 3.0, 2, 2 ** 31 - 1)]
    for acc, m2, cnt in bufs:
        for rule in rules:
            n0 = ctx.launch_count()
            got, n = _select_gpu(ctx, acc, m2, cnt, *rule)
            assert ctx.launch_count() - n0 == 1
            want, wn = select_model(acc, m2, cnt, *rule)
            assert (got == want).all() and n == wn, f"{rule}: {(got != want).sum()} pixels differ"
    assert ctx.last_plan() == plan and ctx.last_render_ms() == ms
    # n_selected may be NULL, and the mask buffer may be uint8
    acc, m2, cnt = bufs[-1]
    mask = torch.full((h, w), 7, dtype=torch.uint8, device="cuda")
    bufs = [_dev(acc), _dev(m2), torch.from_numpy(cnt).cuda()]     # held until the call has run
    torch.cuda.synchronize()
    ctx.adaptive_select_into(*[t.data_ptr() for t in bufs], h, w, 0.02, 0.1, 8, 64, mask.data_ptr(), None)
    ctx.sync()
    assert (_np(mask) == select_model(acc, m2, cnt, 0.02, 0.1, 8, 64)[0]).all()
    ctx.close()


@pytest.mark.gpu
def test_select_past_4_gib(R):
    """20000 x 20000 pixels: 3 * h * w floats of accum and m2 pass 2^32 bytes; a few pixels near the end are read."""
    torch = _torch()
    h = w = 20000
    with R.Context(device=0) as ctx:
        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        m2 = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        counts = torch.full((h, w), -1, dtype=torch.int32, device="cuda")
        rng = np.random.default_rng(9)
        px = np.concatenate([rng.integers(h * w - 10 ** 6, h * w, 2000), rng.integers(0, h * w, 2000)])
        px = np.unique(px)
        c = rng.integers(0, 40, len(px)).astype(np.int32)
        a = (rng.uniform(0, 1, (len(px), 3)) * np.maximum(c, 1)[:, None]).astype(np.float32)
        m = (rng.exponential(3e-3, (len(px), 3)) * np.maximum(c - 1, 1)[:, None]).astype(np.float32)
        idx = torch.from_numpy(px).cuda()
        counts.view(-1)[idx] = torch.from_numpy(c).cuda()
        accum.view(-1, 3)[idx] = torch.from_numpy(a).cuda()
        m2.view(-1, 3)[idx] = torch.from_numpy(m).cuda()
        mask, n = ctx.adaptive_select(accum, m2, counts, 0.02, 0.1, 8, 32)
        want, wn = select_model(a, m, c, 0.02, 0.1, 8, 32)
        assert (_np(mask.view(-1)[idx]) == want).all() and int(n.item()) == wn
        assert int(mask.sum()) == wn
        del accum, m2, counts, mask
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_select_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w = 37, 53
    ctx, _ = _ctx(R, "rgbbox", h, w)
    acc = torch.ones((h, w, 3), device="cuda")
    m2 = torch.ones((h, w, 3), device="cuda")
    cnt = torch.full((h, w), 10, dtype=torch.int32, device="cuda")
    mask = torch.empty((h, w), dtype=torch.bool, device="cuda")
    nan, inf = float("nan"), float("inf")
    cases = [(dict(h=0), "bad image size"), (dict(w=65537), "bad image size"), (dict(accum=None), "required"),
             (dict(m2=None), "required"), (dict(counts=None), "required"), (dict(mask=None), "required"),
             (dict(rel_err=-0.01), "rel_err"), (dict(rel_err=nan), "rel_err"), (dict(rel_err=inf), "rel_err"),
             (dict(mean_floor=-1.0), "mean_floor"), (dict(mean_floor=nan), "mean_floor"), (dict(mean_floor=inf), "mean_floor"),
             (dict(min_count=1), "min_count"), (dict(min_count=-4), "min_count"), (dict(max_count=9), "max_count")]
    good = dict(accum=acc.data_ptr(), m2=m2.data_ptr(), counts=cnt.data_ptr(), h=h, w=w, rel_err=0.02, mean_floor=0.1,
                min_count=10, max_count=64, mask=mask.data_ptr())
    n_sel = torch.empty(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for change, message in cases:
        a = dict(good, **change)
        n0 = ctx.launch_count()
        with pytest.raises(R.RayError, match=message):
            ctx.adaptive_select_into(a["accum"], a["m2"], a["counts"], a["h"], a["w"], a["rel_err"], a["mean_floor"],
                                     a["min_count"], a["max_count"], a["mask"], n_sel.data_ptr())
        assert ctx.launch_count() == n0
        ctx.adaptive_select_into(*[good[k] for k in ("accum", "m2", "counts", "h", "w", "rel_err", "mean_floor",
                                                     "min_count", "max_count", "mask")], n_sel.data_ptr())
        ctx.sync()
        want, wn = select_model(_np(acc), _np(m2), _np(cnt), 0.02, 0.1, 10, 64)
        assert (_np(mask) == want).all() and int(n_sel.item()) == wn, message
    ctx.close()


# ------------------------------------------------------------------------------------------ GPU: the converged loop


@pytest.mark.gpu
@pytest.mark.parametrize("scene,size", [("irreg", 160), ("rgbbox", 128)])
def test_render_converged(R, scene, size):
    torch = _torch()
    h = w = size
    ctx, pr = _ctx(R, scene, h, w)
    min_spp, step, max_spp, rel_err, floor = 4, 4, 64, 0.05, 0.1
    pix, rgb, counts, stats = ctx.render_converged(pr, h, w, rel_err, mean_floor=floor, min_spp=min_spp, step=step,
                                                   max_spp=max_spp, want_rgb=True)
    cnt = _np(counts)
    assert cnt.min() >= min_spp and cnt.max() <= max_spp and ((cnt - min_spp) % step == 0).all()
    assert stats["samples"] == int(cnt.astype(np.int64).sum()) and 1 < stats["rounds"] <= (max_spp - min_spp) // step + 1
    assert len(np.unique(cnt)) >= 2, "an adaptive frame has more than one count"
    pix, rgb = _np(pix), _np(rgb)
    for n in np.unique(cnt):
        p = cnt == n
        want_pix, want_rgb = _one_shot(ctx, pr, h, w, int(n))
        assert (pix[p] == want_pix[p]).all() and bits_differ(rgb[p], want_rgb[p]) == 0, f"count {n}"
    # every pixel that stopped below max_spp is one the rule no longer selects: rebuild accum and m2 by the numpy rule
    colours = _gpu_colours(R, ctx, pr, h, w, int(cnt.max()))
    acc, m2, _ = m2_model(colours, [None], [0])
    for n in np.unique(cnt):
        p = cnt == n
        a, m, _ = m2_model(colours[p][None], [None], [int(n)])
        acc[p], m2[p] = a[0], m[0]
    sel, _ = select_model(acc, m2, cnt, rel_err, floor, min_spp, max_spp - step + 1)
    assert not sel.any(), f"{sel.sum()} pixels are still selected"
    ctx.close()


@pytest.mark.gpu
def test_render_converged_reaches_max_spp_and_rejects_bad_arguments(R):
    ctx, pr = _ctx(R, "irreg", 64, 64)
    pix, counts, stats = ctx.render_converged(pr, 64, 64, 0.0, min_spp=2, step=3, max_spp=11)
    assert (_np(counts) == 11).all() and stats["rounds"] == 4 and stats["samples"] == 64 * 64 * 11
    want_pix, _ = _one_shot(ctx, pr, 64, 64, 11)
    assert (_np(pix) == want_pix).all()
    _, counts, stats = ctx.render_converged(pr, 64, 64, 0.0, min_spp=8, step=8, max_spp=12)
    assert (_np(counts) == 8).all() and stats["rounds"] == 1
    for kw in (dict(min_spp=1), dict(step=0), dict(max_spp=4, min_spp=8)):
        with pytest.raises(ValueError):
            ctx.render_converged(pr, 64, 64, 0.02, **kw)
    with pytest.raises(R.RayError, match="rel_err"):
        ctx.render_converged(pr, 64, 64, -1.0)
    ctx.close()


# ------------------------------------------------------------------------------------------ GPU: ordering, sizes, errors


@pytest.mark.gpu
def test_renders_around_a_loop_plan_and_launch_as_before(R):
    torch = _torch()
    h, w = 250, 250
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")

    def run(with_loop):
        ctx, pr = _ctx(R, "irreg", h, w)
        frames, launches, plans = [], [], []
        for spp in (1, 1, 4, 1, 4):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            launches.append(ctx.launch_count() - n0)
            plans.append(ctx.last_plan())
            frames.append(_np(out))
            if with_loop:
                ctx.render_converged(pr, h, w, 0.05, min_spp=2, step=2, max_spp=8)
        ctx.close()
        return frames, launches, plans

    plain, looped = run(False), run(True)
    assert plain[1] == looped[1] and plain[2] == looped[2]
    assert plain[1][0] > 1 and plain[1][1] == 1, "the learned order is recorded by the first frame and used by the second"
    for a, b in zip(plain[0], looped[0]):
        assert (a == b).all()


@pytest.mark.gpu
def test_torch_stream_and_freeing_the_scene_in_flight(R):
    torch = _torch()
    h, w = 300, 400
    masks, n_adds = [None] + random_masks(h, w, 2, 13), [2, 3, 5]
    ctx, pr = _ctx(R, "rgbbox", h, w)
    want = _var_chain(ctx, pr, h, w, masks, n_adds)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        got = _var_chain(ctx, pr, h, w, masks, n_adds)
    for a, b in zip(want, got):
        assert bits_differ(a.view(np.float32), b.view(np.float32)) == 0, "torch stream"
    ctx.set_stream(None)
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    m2 = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    dmasks = [None if m is None else torch.from_numpy(m).cuda() for m in masks]
    torch.cuda.synchronize()
    for m, n in zip(dmasks, n_adds):
        s, c = SCENES["rgbbox"]()
        pr2 = ctx.prepare_scene(h, w, ctx.scene_from_arrays(s, c))
        ctx.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, pr2, n,
                                     None if m is None else m.data_ptr())
        pr2.free()          # while the call may still be in flight
    ctx.sync()
    assert (_np(counts) == want[2]).all()
    assert bits_differ(_np(accum), want[0]) == 0 and bits_differ(_np(m2), want[1]) == 0
    ctx.close()


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w = 37, 53
    ctx, pr = _ctx(R, "rgbbox", h, w)
    colours = _gpu_colours(R, ctx, pr, h, w, 3)
    want_acc, want_m2, _ = m2_model(colours, [None], [3])
    accum = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    m2 = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")

    class Freed:
        handle = None

    cases = [(dict(n_add=0), "n_add must be >= 1"), (dict(accum=None), "accum_dev is required"),
             (dict(m2=None), "m2_dev is required"), (dict(counts=None), "counts_dev is required"),
             (dict(h=0), "bad image size"), (dict(w=65537), "bad image size"),
             (dict(prepared=Freed()), "invalid prepared scene"), (dict(shard=(1, 2)), "shard set")]
    for change, message in cases:
        a = dict(accum=accum.data_ptr(), m2=m2.data_ptr(), counts=counts.data_ptr(), h=h, w=w, prepared=pr, n_add=3,
                 shard=None)
        a.update(change)
        if a["shard"]:
            ctx.set_shard(*a["shard"])
        n0 = ctx.launch_count()
        with pytest.raises(R.RayError, match=message):
            ctx.render_adaptive_var_into(a["accum"], a["m2"], a["counts"], a["h"], a["w"], a["prepared"], a["n_add"])
        assert ctx.launch_count() == n0
        ctx.set_shard(0, 1)
        counts.zero_()
        torch.cuda.synchronize()
        ctx.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, pr, 3)
        ctx.sync()
        assert bits_differ(_np(accum), want_acc) == 0 and bits_differ(_np(m2), want_m2) == 0, message
    ctx.close()


@pytest.mark.gpu
def test_million_spheres(R):
    h = w = 256
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.scene_random(1 << 20, 1))
        _check_chain(R, ctx, pr, h, w, [None] + random_masks(h, w, 2, 6), [4, 4, 1], "1 M spheres")


@pytest.mark.gpu
def test_largest_frame_sparse_mask(R):
    """2^30 pixels, one in 4096 selected: sum and M2 offsets pass 2^32 bytes; sampled rows against render_into and the
    numpy rule on trace_paths colours."""
    torch = _torch()
    h = w = 32768
    with R.Context(device=0) as ctx:
        pr = ctx.prepare_scene(h, w, ctx.irreg())
        g = torch.Generator(device="cuda").manual_seed(3)
        mask = torch.rand((h, w), device="cuda", generator=g) < 1 / 4096
        rows = [0, 1, h // 2, h - 2, h - 1]
        mask[rows, ::97] = True
        accum = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        m2 = torch.full((h, w, 3), float("nan"), dtype=torch.float32, device="cuda")
        counts = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        pix = torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
        for n in (1, 2):
            ctx.render_adaptive(pr, accum, counts, n, mask=mask, pixels=pix, m2=m2)
        assert int((counts == 3).sum()) == int(mask.sum()) and int((counts[~mask] != 0).sum()) == 0
        m = mask[rows]
        got_m2 = _np(m2[rows][m])
        assert np.isnan(_np(m2[rows][~m])).all()
        del accum, m2
        want = torch.empty((h, w), dtype=torch.int32, device="cuda")
        ctx.render_into(want.data_ptr(), h, w, pr, spp=3)
        ctx.sync()
        assert torch.equal(pix[rows][m], want[rows][m])
        del pix, want, counts
        torch.cuda.empty_cache()
        # the selected pixels of the rows: their samples' colours through trace_paths, for the M2 rule
        rj, ri = np.nonzero(_np(m))
        cam_rays = _pixel_rays(R, pr.info()["camera"], h, w, np.asarray(rows)[rj], ri, 3)
        colours = _np(ctx.trace_paths(pr, _dev(cam_rays.reshape(-1, 6)))[0]).reshape(-1, 1, 3, 3)
        _, want_m2, _ = m2_model(colours, [None], [3])
        assert bits_differ(got_m2, want_m2[:, 0]) == 0
        del mask
        torch.cuda.empty_cache()
