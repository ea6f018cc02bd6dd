"""Ray queries (include/ray_b200.h "ray queries"): caller-supplied rays traced to their closest hit (objs_hit,
ray.fut:76-86) or along their path (ray_colour, ray.fut:126-148).  Every GPU result is compared bit for bit with the CPU
oracle or with a render; NaN (the sky of an all-zero direction) equals any NaN, every other value is compared by its bits."""
import ctypes

import numpy as np
import pytest

import ray_query_oracle as Q   # tests/ray_query_oracle.py: the CPU oracle of the ray queries

# ------------------------------------------------------------------------------------------ helpers


def bits_differ(a, b):
    """Number of float32 values whose bits differ (any NaN equals any NaN)."""
    a = np.ascontiguousarray(a, np.float32).ravel()
    b = np.ascontiguousarray(b, np.float32).ravel()
    assert a.shape == b.shape
    na, nb = np.isnan(a), np.isnan(b)
    return int(((na != nb) | (~na & (a.view(np.uint32) != b.view(np.uint32)))).sum())


def hits_differ(got, want):
    """[n, 8] hit records: the sphere column as int32, the rest by bits."""
    got = np.ascontiguousarray(got, np.float32)
    want = np.ascontiguousarray(want, np.float32)
    bad = int((got[:, 1].view(np.int32) != want[:, 1].view(np.int32)).sum())
    return bad + bits_differ(got[:, [0, 2, 3, 4, 5, 6, 7]], want[:, [0, 2, 3, 4, 5, 6, 7]])


def quantise(rgb):
    """colour_to_pixel (ray.fut:158-162) of float32 [..., 3]."""
    q = (np.float32(255.99) * np.asarray(rgb, np.float32)).astype(np.int32)
    return (q[..., 0] << 16) | (q[..., 1] << 8) | q[..., 2]


def random_rays(spheres, n, seed):
    """Origins uniform in the scene's bounding box expanded by 10 % per side, directions uniform on the sphere."""
    s = np.asarray(spheres, np.float32)
    lo = (s[:, :3] - s[:, 6:7]).min(0)
    hi = (s[:, :3] + s[:, 6:7]).max(0)
    ext = 0.1 * (hi - lo)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo - ext, hi + ext, (n, 3)).astype(np.float32)
    d = rng.standard_normal((n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([o, d], 1), np.float32)


# A hand-built scene with exactly representable answers.  Sphere A (centre 0, radius 1) is second in the caller's array
# and first in Morton order, so a hit on it reports sphere 1; sphere B (centre (0,0,10), radius 1) is first.
TWO_SPHERES = np.array([[0, 0, 10, 0.5, 0.5, 0.5, 1], [0, 0, 0, 0.8, 0.6, 0.4, 1]], np.float32)
TWO_CAM = np.array([0, 0, -20, 0, 0, 0, 60], np.float32)
ALONG_Z = [0, 0, -5, 0, 0, 1]


def two_sphere_cases():
    """(ray, t_min, t_max, expected t, expected sphere, expected p, expected normal) known answers."""
    return [
        (ALONG_Z, 0.0, 1e9, 4.0, 1, (0, 0, -1), (0, 0, -1)),       # front of A: root1 = (5 - 1) / 1
        (ALONG_Z, 5.0, 1e9, -1.0, -1, None, None),                   # t_min > 0.1: the search still takes A at t = 4
                                                                     # (epsilon 0.1, ray.fut:79); re-intersected with
                                                                     # (5, 5) it fails, so B at 14 is not reported
        ([0, 0, -1.0625, 0, 0, 1], 0.0, 1e9, 0.0625, 1, (0, 0, -1), (0, 0, -1)),  # the search skips root 0.0625 <= 0.1
                                                                     # and takes 2.0625; the re-intersection with t_min 0
                                                                     # returns 0.0625 (ray.fut:85)
        (ALONG_Z, 3.0, 3.0, -1.0, -1, None, None),                   # t_max <= t_min: every ray misses
        (ALONG_Z, 0.0, 3.0, -1.0, -1, None, None),                   # shadow-style t_max short of A
        ([0, 0, 12, 0, 0, -1], 0.0, 1e9, 1.0, 0, (0, 0, 11), (0, 0, 1)),          # back of B, from behind
        ([0, 5, 0, 0, 1, 0], 0.0, 1e9, -1.0, -1, None, None),        # away from everything
    ]


def check_two_sphere(out, cases):
    for k, (_, _, _, t, sph, p, nrm) in enumerate(cases):
        rec = out[k]
        assert rec[0] == np.float32(t), (k, rec)
        assert rec[1:2].view(np.int32)[0] == sph, (k, rec)
        if p is not None:
            assert list(rec[2:5]) == list(np.float32(p)), (k, rec)
            assert list(rec[5:8]) == list(np.float32(nrm)), (k, rec)


# ------------------------------------------------------------------------------------------ CPU


def test_hit_struct_is_32_bytes_and_bound(R):
    lib = R.load_library()
    assert ctypes.sizeof(R.Hit) == lib.ray_b200_hit_size() == 32
    bound = set(R.declared_symbols())
    assert {"ray_b200_trace_hits", "ray_b200_trace_paths", "ray_b200_hit_size"} <= bound


@pytest.mark.parametrize("spp", [1, 4])
def test_camera_rays_equal_the_oracle_get_ray(R, spp):
    h, w = 37, 91
    pr = Q.prepare("rgbbox", h, w)
    rays = R.camera_rays(pr.camera(), h, w, spp)
    assert rays.shape == (h, w, spp, 6) and rays.dtype == np.float32
    want = np.array([[[pr.camera_ray(h, w, j, i, s, spp) for s in range(spp)] for i in range(w)] for j in range(h)], np.float32)
    assert bits_differ(rays, want) == 0


@pytest.mark.parametrize("name", ["rgbbox", "irreg"])
def test_oracle_paths_of_camera_rays_equal_oracle_render(R, name):
    h = w = 200
    pr = Q.prepare(name, h, w)
    want, segments = pr.render(h, w)
    rays = R.camera_rays(pr.camera(), h, w).reshape(-1, 6)
    rgb, seg = pr.trace_paths(rays)
    assert int((quantise(rgb).reshape(h, w) != want).sum()) == 0
    assert int(seg.sum()) == segments


@pytest.mark.parametrize("name", ["rgbbox_500", "irreg_500"])
def test_oracle_paths_of_camera_rays_equal_golden_png(R, golden, name):
    pix, _ = golden[name]
    h, w = pix.shape
    pr = Q.prepare(name.split("_")[0], h, w)
    rgb, _ = pr.trace_paths(R.camera_rays(pr.camera(), h, w).reshape(-1, 6))
    assert int((quantise(rgb).reshape(h, w) != pix).sum()) == 0


def test_oracle_two_sphere_known_answers():
    pr = Q.prepare_custom(TWO_SPHERES, TWO_CAM, 64, 64)
    assert list(pr.perm(2)) == [1, 0]
    cases = two_sphere_cases()
    out = np.concatenate([pr.trace_hits(np.array([c[0]], np.float32), c[1], c[2]) for c in cases])
    check_two_sphere(out, cases)
    # paths: the sky straight up is (0.5, 0.7, 1.0) after one segment; max_depth 0 runs no segment
    rgb, seg = pr.trace_paths(np.array([[0, 5, 0, 0, 1, 0]], np.float32))
    assert list(rgb[0]) == [0.5, np.float32(0.7), 1.0] and seg[0] == 1
    rgb, seg = pr.trace_paths(np.array([ALONG_Z], np.float32), max_depth=0)
    assert list(rgb[0]) == [0, 0, 0] and seg[0] == 0


# ------------------------------------------------------------------------------------------ GPU

def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _gpu_case(R, name, h=500, w=500, n=None, seed=1, **ctx_kw):
    ctx = R.Context(device=0, **ctx_kw)
    sc = ctx.scene(name, n=n, seed=seed)
    return ctx, sc, ctx.prepare_scene(h, w, sc)


def _oracle_for(name, h=500, w=500, n=None, seed=1):
    return Q.prepare(name, h, w, n=n, seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgbbox_500", "irreg_500"])
def test_camera_ray_paths_equal_golden(R, golden, name):
    pix, _ = golden[name]
    h, w = pix.shape
    ctx, sc, pr = _gpu_case(R, name.split("_")[0], h, w)
    with ctx:
        rgb, seg = ctx.trace_paths(pr, _dev(R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6)))
        assert int((quantise(rgb.cpu().numpy()).reshape(h, w) != pix).sum()) == 0
        assert int(seg.min()) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(37, 91), (130, 67)])
def test_camera_ray_paths_equal_oracle_odd_sizes(R, hw):
    h, w = hw
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        rays = R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6)
        rgb, seg = ctx.trace_paths(pr, _dev(rays))
        o = _oracle_for("irreg", h, w)
        want_rgb, want_seg = o.trace_paths(rays)
        assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0
        assert int((seg.cpu().numpy() != want_seg).sum()) == 0
        want, _ = o.render(h, w)
        assert int((quantise(rgb.cpu().numpy()).reshape(h, w) != want).sum()) == 0


@pytest.mark.gpu
def test_camera_ray_samples_summed_in_order_equal_render_rgb(R):
    torch = _torch()
    h, w, spp = 64, 96, 4
    ctx, sc, pr = _gpu_case(R, "rgbbox", h, w)
    with ctx:
        pix = torch.empty((h, w), dtype=torch.int32, device="cuda")
        out_rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        ctx.render_into(pix.data_ptr(), h, w, pr, spp=spp, out_rgb_dev=out_rgb.data_ptr())
        ctx.sync()
        rgb, _ = ctx.trace_paths(pr, _dev(R.camera_rays(pr.info()["camera"], h, w, spp).reshape(-1, 6)))
        c = rgb.cpu().numpy().reshape(h, w, spp, 3)
        s = c[:, :, 0]
        for k in range(1, spp):
            s = s + c[:, :, k]
        s = np.float32(1.0 / spp) * s
        assert bits_differ(s, out_rgb.cpu().numpy()) == 0
        assert int((quantise(s) != pix.cpu().numpy()).sum()) == 0


RANDOM_SCENES = [("rgbbox", None, 4096), ("irreg", None, 4096), ("random", 30000, 4096)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_spheres,n", RANDOM_SCENES)
def test_random_rays_equal_oracle(R, name, n_spheres, n):
    ctx, sc, pr = _gpu_case(R, name, n=n_spheres)
    with ctx:
        rays = random_rays(sc.arrays()[0], n, seed=7)
        o = _oracle_for(name, n=n_spheres)
        hits = ctx.trace_hits(pr, _dev(rays))
        got = np.stack([hits["t"].cpu().numpy(), hits["sphere"].cpu().numpy().view(np.float32)], 1)
        got = np.concatenate([got, hits["p"].cpu().numpy(), hits["normal"].cpu().numpy()], 1)
        want = o.trace_hits(rays)
        assert hits_differ(got, want) == 0
        assert (want[:, 0] > 0).mean() > 0.05  # the rays do hit something
        rgb, seg = ctx.trace_paths(pr, _dev(rays))
        want_rgb, want_seg = o.trace_paths(rays)
        assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0
        assert int((seg.cpu().numpy() != want_seg).sum()) == 0


@pytest.mark.gpu
def test_random_rays_on_the_million_sphere_scene(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "random", 2000, 2000, n=1000000)
    with ctx:
        assert pr.info()["smem_nodes"] < pr.info()["n_inner"]
        rays = random_rays(sc.arrays()[0], 65536, seed=11)
        d = _dev(rays)
        hits = torch.empty((rays.shape[0], 8), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()   # the context's own stream is not ordered after torch's
        ctx.trace_hits_into(d.data_ptr(), rays.shape[0], pr, hits.data_ptr())
        rgb, seg = ctx.trace_paths(pr, d)
        sub = slice(0, None, 16)
        o = _oracle_for("random", 2000, 2000, n=1000000)
        assert hits_differ(hits.cpu().numpy()[sub], o.trace_hits(rays[sub])) == 0
        want_rgb, want_seg = o.trace_paths(rays[sub])
        assert bits_differ(rgb.cpu().numpy()[sub], want_rgb) == 0
        assert int((seg.cpu().numpy()[sub] != want_seg).sum()) == 0


@pytest.mark.gpu
def test_two_sphere_known_answers_on_gpu(R):
    with R.Context(device=0) as ctx:
        sc = ctx.scene_from_arrays(TWO_SPHERES, TWO_CAM)
        pr = ctx.prepare_scene(64, 64, sc)
        for c in two_sphere_cases():
            h = ctx.trace_hits(pr, _dev([c[0]]), t_min=c[1], t_max=c[2])
            rec = np.concatenate([h["t"].cpu().numpy(), h["sphere"].cpu().numpy().view(np.float32), h["p"].cpu().numpy()[0],
                                  h["normal"].cpu().numpy()[0]])[None]
            check_two_sphere(rec, [c])


@pytest.mark.gpu
def test_edge_rays_equal_oracle(R):
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        spheres = sc.arrays()[0]
        o = _oracle_for("rgbbox")
        c = spheres[:, :3]
        rad = spheres[:, 6:7]
        rays = [[0, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0], [0, 0, 0, 0, -1, 0], [0, 0, 0, 0, 0, 1],   # all-zero, axis-aligned
                [0, 30, 30, 0, -1, -1], [1, 2, 3, -0.0, 0.0, 1], [0, 0, 0, 1, 1, 0], [-30, -30, -30, 1, 1, 1]]
        rays += [[*(c[k] + rad[k] * np.float32([1, 0, 0])), -1, 0.25, 0.5] for k in range(0, 400, 7)]   # on surfaces
        rays += [[*c[k], 0.3, -1, 0.2] for k in range(3, 400, 11)]                                      # inside spheres
        rays = np.array(rays, np.float32)
        hits = o.trace_hits(rays)
        hit = hits[:, 0] > 0
        # origins at previous hit points, continuing along the reflected-ish direction
        rays = np.concatenate([rays, np.concatenate([hits[hit, 2:5], -rays[hit, 3:6]], 1)]).astype(np.float32)
        g = ctx.trace_hits(pr, _dev(rays))
        got = np.concatenate([g["t"].cpu().numpy()[:, None], g["sphere"].cpu().numpy().view(np.float32)[:, None],
                              g["p"].cpu().numpy(), g["normal"].cpu().numpy()], 1)
        assert hits_differ(got, o.trace_hits(rays)) == 0
        for t_max in (0.05, 0.5, 3.0):   # shadow-style
            g = ctx.trace_hits(pr, _dev(rays), t_min=0.0, t_max=t_max)
            assert bits_differ(g["t"].cpu().numpy(), o.trace_hits(rays, 0.0, t_max)[:, 0]) == 0
        for depth in (0, 1, 2, 50, 200):
            rgb, seg = ctx.trace_paths(pr, _dev(rays), max_depth=depth)
            want_rgb, want_seg = o.trace_paths(rays, max_depth=depth)
            assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0, depth
            assert int((seg.cpu().numpy() != want_seg).sum()) == 0, depth
        assert np.isnan(o.trace_paths(rays[:1])[0]).all()   # the all-zero direction's sky is NaN on both sides


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 33, 1 << 22])
def test_batch_sizes(R, n):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "irreg")
    with ctx:
        rays = random_rays(sc.arrays()[0], max(n, 1), seed=n)[:n]
        d = _dev(rays) if n else torch.empty((0, 6), dtype=torch.float32, device="cuda")
        before = ctx.launch_count()
        rgb, seg = ctx.trace_paths(pr, d)
        hits = ctx.trace_hits(pr, d)
        if n == 0:
            assert ctx.launch_count() == before and rgb.shape == (0, 3)
            return
        assert ctx.launch_count() == before + 2
        assert ctx.last_render_ms() > 0
        sub = slice(None) if n < 1000 else slice(0, None, 997)
        o = _oracle_for("irreg")
        want_rgb, want_seg = o.trace_paths(rays[sub])
        assert bits_differ(rgb.cpu().numpy()[sub], want_rgb) == 0
        assert int((seg.cpu().numpy()[sub] != want_seg).sum()) == 0
        assert bits_differ(hits["t"].cpu().numpy()[sub], o.trace_hits(rays[sub])[:, 0]) == 0


@pytest.mark.gpu
def test_validation_errors_leave_the_context_usable(R):
    torch = _torch()
    ctx, sc, pr = _gpu_case(R, "rgbbox")
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 64, seed=3))
        out = torch.empty((64, 8), dtype=torch.float32, device="cuda")
        rp, op = rays.data_ptr(), out.data_ptr()
        bad = [lambda: ctx.trace_hits_into(rp, -1, pr, op),
               lambda: ctx.trace_hits_into(rp, (1 << 30) + 1, pr, op),
               lambda: ctx.trace_hits_into(None, 64, pr, op),
               lambda: ctx.trace_hits_into(rp, 64, pr, None),
               lambda: ctx.trace_paths_into(rp, 64, pr, None),
               lambda: ctx.trace_hits_into(rp, 64, pr, op, t_min=-1.0),
               lambda: ctx.trace_hits_into(rp, 64, pr, op, t_min=float("nan")),
               lambda: ctx.trace_hits_into(rp, 64, pr, op, t_max=float("inf")),
               lambda: ctx.trace_hits_into(rp, 64, pr, op, t_min=float("inf")),
               lambda: ctx.trace_paths_into(rp, 64, pr, op, max_depth=-1),
               lambda: ctx.trace_paths_into(rp, 64, pr, op, max_depth=65536)]
        for k, call in enumerate(bad):
            with pytest.raises(R.RayError) as e:
                call()
            assert str(e.value), k
        null_scene = type("P", (), {"handle": None})()
        with pytest.raises(R.RayError, match="invalid prepared scene"):
            ctx.trace_hits_into(rp, 64, null_scene, op)
        with pytest.raises(ValueError):
            ctx.trace_hits(pr, rays.double())
        with pytest.raises(ValueError):
            ctx.trace_hits(pr, rays.cpu())
        o = _oracle_for("rgbbox")
        rgb, seg = ctx.trace_paths(pr, rays)
        want_rgb, want_seg = o.trace_paths(rays.cpu().numpy())
        assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0 and (seg.cpu().numpy() == want_seg).all()


@pytest.mark.gpu
def test_torch_stream_pipelined_frames_and_freed_scene(R, golden):
    torch = _torch()
    pix, _ = golden["rgbbox_500"]
    h, w = pix.shape
    with R.Context(device=0) as ctx:
        ctx.set_stream(torch.cuda.current_stream().cuda_stream)
        ctx.set_pipeline(True)
        sc = ctx.rgbbox()
        frame_scene = ctx.prepare_scene(h, w, sc)
        rays = random_rays(sc.arrays()[0], 20000, seed=5)
        o = _oracle_for("rgbbox")
        want_rgb, want_seg = o.trace_paths(rays)
        want_hits = o.trace_hits(rays)
        frames = [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(4)]
        outs = []
        for k in range(4):
            ctx.render_batch([{"prepared": frame_scene, "h": h, "w": w, "out_dev": frames[k].data_ptr()}])
            q = ctx.prepare_scene(h, w, sc)   # a scene used by one query only, freed while the query is in flight
            d = _dev(rays)
            rgb = torch.empty((rays.shape[0], 3), dtype=torch.float32, device="cuda")
            seg = torch.empty((rays.shape[0],), dtype=torch.int32, device="cuda")
            hits = torch.empty((rays.shape[0], 8), dtype=torch.float32, device="cuda")
            ctx.trace_paths_into(d.data_ptr(), rays.shape[0], q, rgb.data_ptr(), seg.data_ptr())
            ctx.trace_hits_into(d.data_ptr(), rays.shape[0], q, hits.data_ptr())
            q.free()
            outs.append((d, rgb, seg, hits))
        ctx.sync()
        torch.cuda.synchronize()
        for k in range(4):
            assert int((frames[k].cpu().numpy() != pix).sum()) == 0, k
            _, rgb, seg, hits = outs[k]
            assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0, k
            assert (seg.cpu().numpy() == want_seg).all(), k
            assert hits_differ(hits.cpu().numpy(), want_hits) == 0, k
        ctx.set_pipeline(False)
        ctx.set_stream(None)


@pytest.mark.gpu
def test_queries_are_invisible_to_renders(R, golden):
    torch = _torch()
    pix, _ = golden["irreg_500"]
    h, w = pix.shape
    ctx, sc, pr = _gpu_case(R, "irreg", h, w)
    with ctx:
        rays = _dev(random_rays(sc.arrays()[0], 50000, seed=9))
        for k in range(3):   # frame 0 records the learned claim order; queries sit between every pair of frames
            img = ctx.render(h, w, pr)
            ctx.trace_hits(pr, rays, t_min=0.5, t_max=100.0)
            ctx.trace_paths(pr, rays, max_depth=7)
            ctx.sync()
            assert int((img.values() != pix).sum()) == 0, k
        out_rgb = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        frame = torch.empty((h, w), dtype=torch.int32, device="cuda")
        ctx.render_into(frame.data_ptr(), h, w, pr, out_rgb_dev=out_rgb.data_ptr())
        ctx.sync()
        assert int((frame.cpu().numpy() != pix).sum()) == 0


PLAN_VARIANTS = [{"wq_k": 1}, {"wq_k": 2}, {"wq_warps": 3}, {"wq_warps": 5}, {"stage_cap": 1024}, {"kernel": "mega"}]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", PLAN_VARIANTS, ids=[",".join(f"{k}={v}" for k, v in d.items()) for d in PLAN_VARIANTS])
def test_plan_variants(R, kw):
    for name in ("rgbbox", "irreg"):
        ctx, sc, pr = _gpu_case(R, name, **kw)
        with ctx:
            rays = random_rays(sc.arrays()[0], 3000, seed=13)
            o = _oracle_for(name)
            rgb, seg = ctx.trace_paths(pr, _dev(rays))
            want_rgb, want_seg = o.trace_paths(rays)
            assert bits_differ(rgb.cpu().numpy(), want_rgb) == 0, name
            assert (seg.cpu().numpy() == want_seg).all(), name
            h = ctx.trace_hits(pr, _dev(rays), t_min=1.0, t_max=200.0)
            assert bits_differ(h["t"].cpu().numpy(), o.trace_hits(rays, 1.0, 200.0)[:, 0]) == 0, name
