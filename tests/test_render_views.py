"""Several views of one prepared scene in one launch (include/ray_b200.h ray_b200_render_views_into).  The contract is
exactness: view v of a call equals, bit for bit, render_into of the prepared scene's spheres prepared again at (h, w)
with cams[v] as their camera.

On the CPU the camera the library makes of a view (make_camera with the call's aspect ratio, the function prepare_scene
uses) is pinned down against the oracle's prepared camera, and the Python argument checks are exercised.  On the GPU
every view is checked bit for bit (NaN-aware) against per-view prepared scenes, on several scenes, view counts, sample
counts, frame sizes and plans, and against the CPU oracle and the golden frames."""
import numpy as np
import pytest

from oracle import pyoracle as O
from ray_query_cases import PLANS, TWO_SPHERES, _np, _torch, bits_differ

SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel writes
INT32_MIN = np.int32(-2 ** 31)


# ------------------------------------------------------------------------------------------ scenes and cameras


def scene_arrays(name):
    """(spheres [n, 7], cam7) of a built-in scene or of 30 000 random spheres."""
    import raytracers_b200 as R
    if name == "random":
        return R.host_scene("random", 30000, 1)
    return R.host_scene(name)


def poses(cam7, n, seed):
    """The scene's own camera, then n - 1 cameras around its look_at: azimuth, elevation, distance, a jittered target
    and a fov in [20, 110] drawn from `seed`."""
    rng = np.random.default_rng(seed)
    c = np.asarray(cam7, np.float32)
    at = c[3:6].astype(np.float64)
    dist = float(np.linalg.norm(c[0:3] - c[3:6]))
    out = [c]
    for _ in range(n - 1):
        az, el, r = rng.uniform(0, 2 * np.pi), rng.uniform(-0.4 * np.pi, 0.45 * np.pi), dist * rng.uniform(0.5, 1.5)
        lf = at + r * np.array([np.cos(el) * np.sin(az), np.sin(el), np.cos(el) * np.cos(az)])
        la = at + rng.normal(0, 0.05 * dist, 3)
        out.append(np.concatenate([lf, la, [rng.uniform(20, 110)]]).astype(np.float32))
    return np.stack(out)


def with_eye(cam7, look_from, look_at):
    c = np.array(cam7, np.float32)
    c[0:3], c[3:6] = look_from, look_at
    return c


# the cameras of tests/test_input_ranges.py whose rays are NaN: looking along vup, and at its own position
TOP_DOWN = ((0, 40, 0), (0, 0, 0))
LOOK_AT_SELF = ((0, 30, 30), (0, 30, 30))


# ------------------------------------------------------------------------------------------ CPU


def _oracle_camera(cam7, h, w):
    return O.Scene.custom(TWO_SPHERES, cam7).prepare(h, w).dump()["cam"]


def test_host_camera_equals_the_oracle(R):
    """The table the library uploads is ray_b200_host_camera's (make_camera, as prepare_scene calls it)."""
    rng = np.random.default_rng(7)
    sizes = [(1, 1), (4, 8), (37, 53), (256, 256), (1000, 1), (3, 700), (500, 500)]
    cams = [scene_arrays(n)[1] for n in ("rgbbox", "irreg", "random")]
    cams += [with_eye(cams[0], *TOP_DOWN), with_eye(cams[1], *TOP_DOWN), with_eye(cams[0], *LOOK_AT_SELF)]
    for fov in (1, 2, 45, 90, 178, 179):
        cams.append(with_eye(np.float32([0, 0, 0, 0, 0, 0, fov]), rng.uniform(-50, 50, 3), rng.uniform(-50, 50, 3)))
    cams += list(poses(cams[1], 20, 3))
    nan_seen = 0
    for c in cams:
        for h, w in sizes:
            got, want = R.host_camera(c, h, w), _oracle_camera(c, h, w)
            assert bits_differ(got, want) == 0, (c, h, w)
            nan_seen += bool(np.isnan(want).any())
    assert nan_seen == 3 * len(sizes), "the NaN cameras are there to give NaN rays"


def test_camera_table_argument_checks(R):
    want = np.float32([[0, 1, 2, 3, 4, 5, 60], [6, 7, 8, 9, 10, 11, 90]])
    for ok in (want, want.astype(np.float64), want.tolist(), _torch().from_numpy(want)):
        got = R.camera_table(ok)
        assert got.dtype == np.float32 and got.flags.c_contiguous and (got == want).all()
    assert R.camera_table(want[::-1]).flags.c_contiguous
    for bad in (want[0], want[:, :6], want[None], want.astype(np.int32), [[1] * 7], np.zeros((2, 8), np.float32)):
        with pytest.raises(ValueError):
            R.camera_table(bad)


# ------------------------------------------------------------------------------------------ GPU helpers


def per_view(ctx, spheres, cams, h, w, spp):
    """(pixels [V, h, w], rgb [V, h, w, 3]) of render_into, one scene prepared at (h, w) per camera."""
    torch = _torch()
    pix = torch.full((len(cams), h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((len(cams), h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    for v, c in enumerate(cams):
        sc = ctx.scene_from_arrays(spheres, c)
        pr = ctx.prepare_scene(h, w, sc)
        ctx.render_into(pix[v].data_ptr(), h, w, pr, spp=spp, out_rgb_dev=rgb[v].data_ptr())
        pr.free()
        sc.free()
    ctx.sync()
    return _np(pix), _np(rgb)


def views(ctx, pr, cams, h, w, spp):
    """(pixels, rgb) of one render_views_into call into sentinel-filled buffers."""
    torch = _torch()
    pix = torch.full((len(cams), h, w), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.full((len(cams), h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    torch.cuda.synchronize()
    ctx.render_views_into(pr, cams, h, w, spp, pix.data_ptr(), rgb.data_ptr())
    ctx.sync()
    return _np(pix), _np(rgb)


def check(got, want, what):
    pix, rgb = got
    wpix, wrgb = want
    assert pix.shape == wpix.shape, what
    bad = pix != wpix
    assert not bad.any(), f"{what}: {int(bad.sum())} pixels differ, in views {sorted(set(np.nonzero(bad)[0].tolist()))}"
    assert bits_differ(rgb, wrgb) == 0, f"{what}: float framebuffer"


def _prepared(ctx, spheres, cam, h, w):
    return ctx.prepare_scene(h, w, ctx.scene_from_arrays(spheres, cam))


# ------------------------------------------------------------------------------------------ GPU: exactness

SIZES = [(1, 1), (4, 8), (37, 53), (256, 256)]
VIEW_COUNTS = [1, 2, 3, 6, 64]


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 2, 7, 64])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg", "random"])
def test_views_equal_prepared_renders(R, scene, spp):
    """Every view count and frame size, each view against render_into of a scene prepared with its camera.  The views
    call uses a scene prepared with some other camera at another size: the BVH does not depend on either."""
    spheres, cam = scene_arrays(scene)
    cams = poses(cam, 64, spp)
    rng = np.random.default_rng(spp)
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, spheres, cams[5], 17, 29)
        for h, w in SIZES:
            want = per_view(ctx, spheres, cams, h, w, spp)
            for n in VIEW_COUNTS:
                pick = np.sort(rng.choice(64, n, replace=False)) if n < 64 else np.arange(64)
                check(views(ctx, pr, cams[pick], h, w, spp), (want[0][pick], want[1][pick]), f"{h}x{w} V={n} {pick}")


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(4, 8), (37, 53)])
@pytest.mark.parametrize("scene", ["rgbbox", "irreg"])
def test_small_frames_equal_the_oracle(R, scene, h, w):
    """Moved cameras and NaN cameras between them against the CPU oracle's render of the custom scene."""
    spheres, cam = scene_arrays(scene)
    cams = np.concatenate([poses(cam, 3, 11), [with_eye(cam, *TOP_DOWN)], poses(cam, 2, 12)[1:],
                           [with_eye(cam, *LOOK_AT_SELF)]])
    for spp in (1, 3):
        want_pix, want_rgb = [], []
        for c in cams:
            p, rgb, _ = O.Scene.custom(spheres, c).prepare(h, w).render(h, w, spp, want_rgb=True)
            want_pix.append(p)
            want_rgb.append(rgb)
        with R.Context(device=0) as ctx:
            pr = _prepared(ctx, spheres, cam, h, w)
            check(views(ctx, pr, cams, h, w, spp), (np.stack(want_pix), np.stack(want_rgb)), f"spp={spp}")


@pytest.mark.gpu
def test_nan_camera_views_do_not_touch_their_neighbours(R):
    h, w, spp = 61, 83, 4
    spheres, cam = scene_arrays("irreg")
    normal = poses(cam, 3, 5)
    cams = np.stack([normal[0], with_eye(cam, *TOP_DOWN), normal[1], with_eye(cam, *LOOK_AT_SELF), normal[2]])
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        got = views(ctx, pr, cams, h, w, spp)
        check(got, per_view(ctx, spheres, cams, h, w, spp), "NaN cameras")
        # alone, the normal views give the same frames
        check(views(ctx, pr, normal, h, w, spp), (got[0][[0, 2, 4]], got[1][[0, 2, 4]]), "without the NaN views")
    assert (got[0][[1, 3]] == np.int32(-2 ** 31)).all(), "a NaN camera quantises to INT32_MIN channels"
    assert not (got[0][[0, 2, 4]] == INT32_MIN).any()


@pytest.mark.gpu
def test_golden_camera_among_other_views(R, golden):
    for name, (pixels, meta) in golden.items():
        h, w = meta["shape"]
        spheres, cam = scene_arrays(name.split("_")[0])
        cams = poses(cam, 4, 9)[[1, 0, 2, 3]]        # the scene's own camera second
        with R.Context(device=0) as ctx:
            pr = _prepared(ctx, spheres, cams[2], 100, 300)
            pix, _ = views(ctx, pr, cams, h, w, 1)
        assert (pix[1] == pixels).all(), name
        assert not (pix[0] == pixels).all(), f"{name}: the other views are other frames"


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS + [{"wq_packet": 24}, {"wq_packet": 0}, {"wq_spread": 0}, {"wq_spread": 1},
                                          {"heavy_first": -1}, {"heavy_first": 4}, {"kernel": "mega"}], ids=str)
def test_every_plan(R, plan):
    h, w = 61, 83
    spheres, cam = scene_arrays("irreg")
    cams = poses(cam, 6, 21)
    with R.Context(device=0) as ref:
        want = {spp: per_view(ref, spheres, cams, h, w, spp) for spp in (1, 16)}
    with R.Context(device=0, **plan) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        for spp in (1, 16):
            check(views(ctx, pr, cams, h, w, spp), want[spp], f"{plan} spp={spp}")


@pytest.mark.gpu
def test_million_spheres(R, oracle):
    """8 views of the 1 M-sphere scene against per-view prepared scenes, and two of them on oracle rows."""
    h = w = 256
    spp, rows = 2, (37, 64)
    spheres, cam = R.host_scene("random", 1000000, 1)
    cams = poses(cam, 8, 4)
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        got = views(ctx, pr, cams, h, w, spp)
        check(got, per_view(ctx, spheres, cams, h, w, spp), "1 M spheres")
    for v in (0, 5):
        want, _, _ = oracle.Scene.custom(spheres, cams[v]).prepare(h, w).render(h, w, spp, row_start=rows[0], row_step=rows[1])
        r = np.arange(rows[0], h, rows[1])
        assert (got[0][v][r] == want[r]).all(), v
    assert len(np.unique(got[0])) > 1000


# ------------------------------------------------------------------------------------------ GPU: plan, streams, errors


@pytest.mark.gpu
def test_renders_around_views_plan_and_launch_as_before(R):
    """A render's frame and launches do not depend on views calls in between (the learned order stays the scene's)."""
    torch = _torch()
    h, w = 250, 250
    spheres, cam = scene_arrays("irreg")
    out = torch.empty((h, w), dtype=torch.int32, device="cuda")
    cams = poses(cam, 3, 2)

    def run(with_views):
        ctx = R.Context(device=0)
        pr = _prepared(ctx, spheres, cam, h, w)
        frames, launches = [], []
        for spp in (1, 1, 4, 1, 4):
            n0 = ctx.launch_count()
            ctx.render_into(out.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            launches.append(ctx.launch_count() - n0)
            frames.append(_np(out))
            if with_views:
                for s in (1, 4):
                    n0 = ctx.launch_count()
                    ctx.render_views(pr, cams, h, w, s)
                    assert ctx.launch_count() - n0 == 1, "one launch per call"
                    assert ctx.last_render_ms() > 0
        ctx.close()
        return frames, launches

    plain, viewed = run(False), run(True)
    assert plain[1] == viewed[1]
    assert plain[1][0] > 1 and plain[1][1] == 1, "the learned order is recorded by the first frame and used by the second"
    for a, b in zip(plain[0], viewed[0]):
        assert (a == b).all()


@pytest.mark.gpu
def test_heavy_first_probe(R):
    """With the heavy-first order on, a views call at spp > 1 probes its tiles with their own cameras, as render_into
    probes a frame: the same launches, the same frames."""
    h, w = 123, 157
    spheres, cam = scene_arrays("irreg")
    cams = poses(cam, 5, 8)
    want = per_view(R.Context(device=0), spheres, cams, h, w, 8)
    with R.Context(device=0, heavy_first=4) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        torch = _torch()
        scratch = torch.empty((h, w), dtype=torch.int32, device="cuda")
        for spp in (1, 8):
            n0 = ctx.launch_count()
            ctx.render_into(scratch.data_ptr(), h, w, pr, spp=spp)
            ctx.sync()
            n_into = ctx.launch_count() - n0
            n0 = ctx.launch_count()
            got = views(ctx, pr, cams, h, w, spp)
            assert ctx.launch_count() - n0 == n_into, spp
        assert n_into == 3, "probe, sort, frame"
        check(got, want, "heavy-first")


@pytest.mark.gpu
def test_torch_stream_reused_cameras_and_freeing_the_scene_in_flight(R):
    torch = _torch()
    h, w, spp = 300, 400, 4
    spheres, cam = scene_arrays("rgbbox")
    cams = poses(cam, 4, 6)
    with R.Context(device=0) as ctx:
        want = per_view(ctx, spheres, cams, h, w, spp)
        pr = _prepared(ctx, spheres, cam, h, w)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            pix, rgb = ctx.render_views(pr, cams, h, w, spp, want_rgb=True)
        check((_np(pix), _np(rgb)), want, "torch stream")
        ctx.set_stream(None)
        pix = torch.full((4, h, w), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        table = cams.copy()
        for v in range(2):
            pr2 = _prepared(ctx, spheres, cam, 50, 50)
            ctx.render_views_into(pr2, table[2 * v:2 * v + 2], h, w, spp, pix[2 * v].data_ptr())
            pr2.free()                      # while the call may still be in flight
            table[2 * v:2 * v + 2] = np.nan  # and the cameras are the caller's again
        ctx.sync()
        assert (_np(pix) == want[0]).all()


@pytest.mark.gpu
def test_errors_leave_the_context_usable(R):
    torch = _torch()
    h, w, spp = 37, 53, 3
    spheres, cam = scene_arrays("rgbbox")
    cams = poses(cam, 3, 1)
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        want = views(ctx, pr, cams, h, w, spp)
        pix = torch.empty((3, h, w), dtype=torch.int32, device="cuda")

        class Freed:
            handle = None

        def good():
            ctx.render_views_into(pr, cams, h, w, spp, pix.data_ptr())
            ctx.sync()
            assert (_np(pix) == want[0]).all()

        lib = ctx.lib
        c = np.ascontiguousarray(cams, np.float32)
        big = np.repeat(cams[:1], 65, 0)          # 65 x 2^19 tiles of 4096^2 > 2^25
        cases = [
            (lambda: ctx.render_views_into(pr, cams[:0], h, w, spp, pix.data_ptr()), "n_views must be >= 1"),
            (lambda: ctx._check(lib.ray_b200_render_views_into(ctx.handle, pr.handle, c.ctypes.data, -3, h, w, spp,
                                                               pix.data_ptr(), None)), "n_views must be >= 1"),
            (lambda: ctx._check(lib.ray_b200_render_views_into(ctx.handle, pr.handle, None, 3, h, w, spp, pix.data_ptr(),
                                                               None)), "cams7_host is required"),
            (lambda: ctx.render_views_into(pr, cams, h, w, spp, None), "out_pix_dev is required"),
            (lambda: ctx.render_views_into(pr, cams, 0, w, spp, pix.data_ptr()), "bad image size"),
            (lambda: ctx.render_views_into(pr, cams, h, 65537, spp, pix.data_ptr()), "bad image size"),
            (lambda: ctx.render_views_into(pr, cams, h, w, 0, pix.data_ptr()), "spp must be >= 1"),
            (lambda: ctx.render_views_into(Freed(), cams, h, w, spp, pix.data_ptr()), "invalid prepared scene"),
            (lambda: ctx.render_views_into(pr, big, 4096, 4096, 1, pix.data_ptr()), "exceed 2\\^30 padded pixels"),
        ]
        for call, message in cases:
            with pytest.raises(R.RayError, match=message):
                call()
            good()
        ctx.set_shard(1, 2)
        with pytest.raises(R.RayError, match="shard set"):
            ctx.render_views_into(pr, cams, h, w, spp, pix.data_ptr())
        ctx.set_shard(0, 1)
        good()
        for bad in (torch.from_numpy(cams).cuda(), cams[0], cams[:, :6], cams.astype(np.int64), [[1, 2, 3]]):
            with pytest.raises(ValueError):
                ctx.render_views(pr, bad, h, w)
            good()


@pytest.mark.gpu
def test_outputs_past_4_gib(R):
    """4 views of 16384^2 = 2^30 pixels: the pixel offsets pass 2^32 bytes, the float frames 12 GiB."""
    torch = _torch()
    h = w = 16384
    spheres, cam = scene_arrays("irreg")
    cams = poses(cam, 4, 30)[[1, 2, 0, 3]]
    with R.Context(device=0) as ctx:
        pr = _prepared(ctx, spheres, cam, h, w)
        pix, rgb = ctx.render_views(pr, cams, h, w, 1, want_rgb=True)
        want_pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
        want_rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        for v in range(4):
            pv = _prepared(ctx, spheres, cams[v], h, w)
            torch.cuda.synchronize()
            ctx.render_into(want_pix.data_ptr(), h, w, pv, spp=1, out_rgb_dev=want_rgb.data_ptr())
            ctx.sync()
            pv.free()
            assert torch.equal(pix[v], want_pix), v
            a, b = rgb[v], want_rgb
            differ = (a.view(torch.int32) != b.view(torch.int32)) & ~(a.isnan() & b.isnan())
            assert int(differ.sum()) == 0, v
        del pix, rgb, want_pix, want_rgb
        torch.cuda.empty_cache()
