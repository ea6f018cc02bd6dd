"""Helpers and cases shared by the ray-query tests (test_ray_queries.py, test_occlusion.py, test_multi_hits.py and
test_limits.py): result comparison, random and shadow rays, the two-sphere scene, the GPU set-up, and the intervals,
plans and scenes the query kinds are all checked on.  Not a test module."""
import numpy as np

GiB = 1 << 30
T24 = np.float32(1 << 24)

# ------------------------------------------------------------------------------------------ comparison and rays


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


def max_hit_t(spheres, rays):
    """An upper bound of every t at which a ray can meet a sphere: a hit point lies on some sphere, so
    t * |d| <= |o - c| + r for that sphere.  Rays with d = 0 never hit (their discriminant is 0)."""
    s = np.asarray(spheres, np.float64)
    r = np.asarray(rays, np.float64)
    dist = np.linalg.norm(r[:, None, :3] - s[None, :, :3], axis=2).max(1) + s[:, 6].max()
    dn = np.linalg.norm(r[:, 3:6], axis=1)
    ok = dn > 0
    return float((dist[ok] / dn[ok]).max()) if ok.any() else 0.0


def light_above(spheres):
    """A point light above the middle of the scene's bounding box, one box height above its top."""
    s = np.asarray(spheres, np.float32)
    lo = (s[:, :3] - s[:, 6:7]).min(0)
    hi = (s[:, :3] + s[:, 6:7]).max(0)
    return np.float32([(lo[0] + hi[0]) / 2, hi[1] + (hi[1] - lo[1]), (lo[2] + hi[2]) / 2])


def segment_rays(points, target):
    """Point-to-point visibility rays: origin = point, direction = target - point (not normalised), so that the
    interval (1e-4, 1 - 1e-4) covers the open segment."""
    p = np.asarray(points, np.float32)
    return np.ascontiguousarray(np.concatenate([p, np.asarray(target, np.float32)[None] - p], 1), np.float32)


SEGMENT = (1e-4, 1 - 1e-4)


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


def _np(t):
    return t.cpu().numpy()


INTERVALS = [(0.0, 1e9), (0.1, 1e9), (1.0, 100.0), (2.5, 1e9), (40.0, 7.0)]
RANDOM_SCENES = [("rgbbox", None), ("irreg", None), ("random", 30000)]


def _shadow_case(R, ctx, sc, pr, h, w):
    """Camera rays through trace_hits, then segments from every hit point to the light."""
    hits = ctx.trace_hits(pr, _dev(R.camera_rays(pr.info()["camera"], h, w).reshape(-1, 6)))
    t = _np(hits["t"])
    return segment_rays(_np(hits["p"])[t >= 0], light_above(sc.arrays()[0]))


PLANS = [{}, {"wq_k": 1}, {"wq_k": 2}, {"wq_warps": 3}, {"wq_warps": 5}, {"stage_cap": 1024}, {"wq_low": -1},
         {"wq_low": 64}, {"wq_ncap": 256}]
