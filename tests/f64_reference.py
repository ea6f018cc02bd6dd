"""A float64 restatement of the reference's semantics (ray.fut, bvh.fut, prim.fut) and of the extensions' contracts in
include/ray_b200.h: camera, spp sample offsets, closest hit with the bvh_fold culling of the fixed-sweep refit's boxes,
ray_colour, the occlusion and multi-hit queries, and quantisation.  TEST INFRASTRUCTURE ONLY; not a test module.

It is written from the reference and the header alone, independently of oracle/oracle.cpp and of the product, and
takes only the tree topology (left, right, parent, perm of host_lbvh) from the library; the boxes are refitted here.

f32 and f64 legitimately disagree near ties, grazing hits, interval ends, scatter-sign flips, stale-box slack and
quantisation boundaries, so every answer comes with a margin: the smallest relative distance of any deciding quantity
from the boundary where the f32 answer could flip.  A sample (or ray) is *judged* when its margin exceeds TAU and, for
paths, when directions perturbed by about 1e-5 give the same spheres and colours.  Comparisons assert agreement on
judged samples only, and a floor on the judged fraction keeps them from judging nothing.
"""
import numpy as np

EPS = 0.1                      # scene_epsilon (ray.fut:3)
TAU = 1e-5                     # a margin below this is a near-tie: the sample is not judged
PERTURB = 1e-5                 # relative size of the two perturbations of a path's primary direction
COLOUR_TOL = 2e-4              # the largest colour error estimate a judged sample may have, relative to max(1, |c|)
QUANT_TAU = 0.002              # distance of 255.99 c from an integer below which a pixel is not judged
OFFSET_X, OFFSET_Y = np.float32(0.7548776662), np.float32(0.5698402909)
SKY = np.array([0.5, 0.7, 1.0])
U32 = 2.0 ** -24               # the unit roundoff of f32
MUTANTS = ("aspect_h_over_w", "v_from_j", "offsets_s_plus_1", "sky_from_x", "no_stale_culling", "no_perm",
           "reintersect_from_eps", "offsets_in_f64", "welford_old_mean", "select_without_count",
           "gbuffer_depth_last_sample", "gbuffer_id_in_leaf_order", "gbuffer_miss_albedo_black")
_PAIR_BUDGET = 1 << 21          # rays x spheres per chunk of the dense discriminant pass (8 f64 arrays of this size)


def _dot(a, b):
    return (a * b).sum(-1)


def _normalise(v):
    with np.errstate(invalid="ignore", divide="ignore"):
        return v / np.sqrt(_dot(v, v))[..., None]


# ------------------------------------------------------------------------------------------ camera and samples


def make_camera(cam7, h, w, aspect=None):
    """camera look_from look_at (0,1,0) fov (w/h) (ray.fut:93-107, 243-244): origin, llc, horizontal, vertical."""
    c = np.asarray(cam7, np.float32).astype(np.float64)
    look_from, look_at, fov = c[0:3], c[3:6], c[6]
    aspect = w / h if aspect is None else aspect
    half_h = np.tan(fov * np.pi / 180.0 / 2.0)
    half_w = aspect * half_h
    with np.errstate(invalid="ignore", divide="ignore"):
        wv = _normalise(look_from - look_at)
        u = _normalise(np.cross([0.0, 1.0, 0.0], wv))
        v = np.cross(wv, u)
    llc = look_from - half_w * u - half_h * v - wv
    return look_from, llc, 2.0 * half_w * u, 2.0 * half_h * v


def sample_offsets(s, mutant=None):
    """(ox_s, oy_s) = frac(f32(s) * 0.7548776662f), frac(f32(s) * 0.5698402909f) for int64 indices s, as f64
    (include/ray_b200.h, spp semantics).  The rule is discrete: f32(s), the f32 product, its floor and the difference
    are each one exact or correctly rounded step, so restating it in f32 is the rule itself, not an approximation of
    it.  From 2^21 / c on the offsets are quarters and halves, and from 2^23 / c on they are 0."""
    s = np.asarray(s, np.int64) + (1 if mutant == "offsets_s_plus_1" else 0)
    if mutant == "offsets_in_f64":   # frac(s * c) in f64: right to about 3e-6 below 2^16, wrong by up to 0.99 at 2^21 / c on
        s = s.astype(np.float64)
        return np.modf(s * 0.7548776662)[0], np.modf(s * 0.5698402909)[0]
    sf = s.astype(np.float32)
    a, b = sf * OFFSET_X, sf * OFFSET_Y
    return (a - np.floor(a)).astype(np.float64), (b - np.floor(b)).astype(np.float64)


def primary_rays(cam7, h, w, j, i, s, mutant=None):
    """Sample s of pixel (row j, column i): u = (i + ox_s) / W, v = (H - j + oy_s) / H, get_ray (ray.fut:109-114)."""
    ox, oy = sample_offsets(s, mutant)
    return offset_rays(cam7, h, w, j, i, ox, oy, mutant)


def offset_rays(cam7, h, w, j, i, ox, oy, mutant=None):
    """primary_rays with the sample offsets (ox, oy) given."""
    aspect = h / w if mutant == "aspect_h_over_w" else None
    origin, llc, hor, ver = make_camera(cam7, h, w, aspect)
    j = np.asarray(j, np.float64)
    u = (np.asarray(i, np.float64) + ox) / w
    v = ((j if mutant == "v_from_j" else h - j) + oy) / h
    d = llc + u[:, None] * hor + v[:, None] * ver - origin
    return np.broadcast_to(origin, d.shape).copy(), d


def _perturbed(D):
    """The two directions D perturbed by PERTURB relative, orthogonally to D and to each other."""
    dn = np.sqrt(_dot(D, D))[:, None]
    e1 = np.cross(D, [0.0, 0.0, 1.0])
    e1 = np.where((np.abs(_dot(e1, e1)) < 1e-12 * dn[:, 0] ** 2)[:, None], np.cross(D, [1.0, 0.0, 0.0]), e1)
    e1 = _normalise(e1)
    e2 = _normalise(np.cross(D, e1))
    return D + PERTURB * dn * e1, D + PERTURB * dn * e2


# ------------------------------------------------------------------------------------------ quantisation


def quantise(c):
    """colour_to_pixel (ray.fut:158-162) by the header's rule: each channel 255.99 c truncated, INT32_MIN where that is
    NaN or outside [-2^31, 2^31), packed with 32-bit wrapping shifts.  Returns (int32 pixels, margin): the margin is
    the smallest distance of 255.99 c from a step of the truncation (a nonzero integer) over the channels.  A NaN
    channel (from a NaN camera ray) is NaN on both sides and has no step."""
    with np.errstate(invalid="ignore", over="ignore"):
        v = 255.99 * np.asarray(c, np.float64)
        ok = (v >= -2.0 ** 31) & (v < 2.0 ** 31)
        q = np.where(ok, np.trunc(np.where(ok, v, 0)), -2.0 ** 31).astype(np.int64) & 0xFFFFFFFF
        frac = np.where(np.abs(v) < 1, 1 - np.abs(v), np.abs(v - np.round(v)))
    margin = np.where(np.isnan(frac), np.inf, frac).min(-1)
    pix = ((q[..., 0] << 16) | (q[..., 1] << 8) | q[..., 2]) & 0xFFFFFFFF
    return pix.astype(np.uint32).view(np.int32), margin


# ------------------------------------------------------------------------------------------ the BVH's boxes


def refit_boxes(leaf_spheres, left, right, sweeps):
    """bvh_mk's boxes (bvh.fut:44-58) in f32: `sweeps` Jacobi sweeps of enclosing (prim.fut:38-45) from zero boxes over
    the given topology (inner i -> i, leaf i -> ~i), leaf boxes sphere_aabb (ray.fut:28-30); sweeps=None runs to the
    fixpoint (every box the union of its children's).  Returns (boxes, leaf boxes)."""
    L = np.asarray(leaf_spheres, np.float32)
    leaf = np.concatenate([L[:, :3] - L[:, 6:7], L[:, :3] + L[:, 6:7]], 1)
    boxes = np.zeros((len(left), 6), np.float32)

    def child(src, c):
        return np.where((c >= 0)[:, None], src[np.maximum(c, 0)], leaf[np.maximum(~c, 0)])

    k = 0
    while sweeps is None or k < sweeps:
        a, b = child(boxes, left), child(boxes, right)
        new = np.concatenate([np.fmin(a[:, :3], b[:, :3]), np.fmax(a[:, 3:], b[:, 3:])], 1).astype(np.float32)
        if sweeps is None and np.array_equal(new.view(np.uint32), boxes.view(np.uint32)):
            break
        boxes, k = new, k + 1
    return boxes, leaf


def refit_sweeps(n):
    """t32 (f32.log2 (f32.i64 n)) + 2 (bvh.fut:47)."""
    return int(np.trunc(np.log2(np.float32(n)))) + 2


def _root_scale(a, b, sq, oc2r2):
    """The magnitude a root's f32 error is relative to: the terms of (-b -+ sqrt(disc)) / a, and the cancellation of
    c = |oc|^2 - r^2 (oc2r2 = |oc|^2 + r^2), which decides roots near 0 such as a ray leaving a sphere's surface."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return (np.abs(b) + sq) / a + oc2r2 / (np.abs(b) + sq + 1e-30)


def _slab(box, o, d, lo, hi):
    """aabb_hit (ray.fut:53-70) in f64 with NaN-ignoring max / min, as a signed relative slack: > 0 iff the box passes."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = 1.0 / d
        t0 = (box[:, :3] - o) * inv
        t1 = (box[:, 3:] - o) * inv
        neg = inv < 0
        ta, tb = np.where(neg, t1, t0), np.where(neg, t0, t1)
        tmin, tmax = lo.copy(), hi.copy()
        for k in range(3):
            tmin = np.fmax(ta[:, k], tmin)
            tmax = np.fmin(tb[:, k], tmax)
        return (tmax - tmin) / np.maximum(np.maximum(np.abs(tmin), np.abs(tmax)), 1e-30)


# ------------------------------------------------------------------------------------------ the reference


class Reference:
    """A prepared scene in f64: spheres float32[n][7] in the caller's order and the LBVH topology of host_lbvh
    (dict with left, right, parent, perm).  `mutant` (one of MUTANTS) makes a deliberately wrong variant."""

    def __init__(self, spheres, topo, cam7=None, mutant=None):
        assert mutant is None or mutant in MUTANTS, mutant
        self.mutant = mutant
        self.spheres = np.ascontiguousarray(spheres, np.float32).reshape(-1, 7)
        self.cam7 = None if cam7 is None else np.asarray(cam7, np.float32)
        n = self.spheres.shape[0]
        self.perm = np.asarray(topo["perm"], np.int64)
        self.left = np.asarray(topo["left"], np.int64)
        self.right = np.asarray(topo["right"], np.int64)
        self.parent = np.asarray(topo["parent"], np.int64)
        L = self.spheres[self.perm]                    # bvh.L: the spheres in Morton order
        self.sweeps = refit_sweeps(n)
        self.boxes, self.leaf_boxes = refit_boxes(L, self.left, self.right, self.sweeps)
        again, _ = refit_boxes(L, self.left, self.right, self.sweeps + 1)
        self.stale = (self.boxes.view(np.uint32) != again.view(np.uint32)).any(1)
        self.fixpoint_boxes, _ = refit_boxes(L, self.left, self.right, None)
        self.cull_boxes = (self.fixpoint_boxes if mutant == "no_stale_culling" else self.boxes).astype(np.float64)
        self.C = L[:, :3].astype(np.float64)
        self.col = L[:, 3:6].astype(np.float64)
        self.rad = L[:, 6].astype(np.float64)
        self.rr = self.rad * self.rad
        self.leaf_parent = np.full(n, -1, np.int64)
        for ch in (self.left, self.right):
            k = np.nonzero(ch < 0)[0]
            self.leaf_parent[~ch[k]] = k
        # geometry id: leaves with bit-identical centre and radius give bit-identical f32 roots, so their tie is exact
        _, self.geom = np.unique(np.ascontiguousarray(L[:, [0, 1, 2, 6]]).view(np.uint32), axis=0, return_inverse=True)
        self.geom = self.geom.ravel()

    # -------------------------------------------------------------------- ray x sphere pairs

    def _pairs(self, O, D, lo, hi):
        """Every (ray, leaf) pair whose line comes near the sphere with a root near (lo, hi) of the ray, with the
        sphere_hit quantities (ray.fut:32-51) in f64: dict of ray, leaf, a, b, disc, r1, r2, rs (root scale)."""
        n = self.C.shape[0]
        chunk = max(1, _PAIR_BUDGET // n)
        CD2 = _dot(self.C, self.C) - self.rr
        ri, li = [], []
        for s in range(0, len(O), chunk):
            o, d = O[s:s + chunk], D[s:s + chunk]
            a = _dot(d, d)[:, None]
            b = _dot(o, d)[:, None] - d @ self.C.T
            c = _dot(o, o)[:, None] - 2.0 * (o @ self.C.T) + CD2[None, :]
            disc = b * b - a * c
            keep = disc > -2 * TAU * (b * b + np.abs(a * c)) - 1e-30   # robust misses are dropped
            r, l = np.nonzero(keep)
            ri.append(r + s)
            li.append(l)
        ri = np.concatenate(ri) if ri else np.zeros(0, np.int64)
        li = np.concatenate(li) if li else np.zeros(0, np.int64)
        oc = O[ri] - self.C[li]
        d = D[ri]
        a = _dot(d, d)
        b = _dot(oc, d)
        c = _dot(oc, oc) - self.rr[li]
        disc = b * b - a * c
        with np.errstate(divide="ignore", invalid="ignore"):
            sq = np.sqrt(np.maximum(disc, 0.0))
            r1, r2 = (-b - sq) / a, (-b + sq) / a
            rs = _root_scale(a, b, sq, _dot(oc, oc) + self.rr[li])
            dm = np.abs(disc) / (b * b + np.abs(a * c))
        keep = (a > 0) & (r2 > lo[ri] - 0.01 * (rs + np.abs(lo[ri])) - 1e-6) & (r1 < hi[ri] + 0.01 * (rs + np.abs(hi[ri])))
        P = dict(ray=ri, leaf=li, a=a, b=b, disc=disc, r1=r1, r2=r2, rs=rs, dm=np.nan_to_num(dm, nan=0.0))
        return {k: v[keep] for k, v in P.items()}

    def _reached(self, P, O, D, lo, hi):
        """bvh_fold's culling (bvh.fut:61-84): a leaf is reached iff every inner ancestor's box passes aabb_hit on
        (lo, hi).  Returns the smallest signed slack over the ancestors' tests (> 0 iff reached)."""
        ri = P["ray"]
        node = self.leaf_parent[P["leaf"]].copy()
        g = np.full(len(ri), np.inf)
        act = np.nonzero(node >= 0)[0]
        while act.size:
            r = ri[act]
            g[act] = np.minimum(g[act], _slab(self.cull_boxes[node[act]], O[r], D[r], lo[r], hi[r]))
            node[act] = self.parent[node[act]]
            act = act[node[act] >= 0]
        return g

    @staticmethod
    def _rel(x, bound, scale):
        with np.errstate(invalid="ignore"):
            return np.nan_to_num(np.abs(x - bound) / (scale + np.abs(bound) + 1e-30), nan=0.0)

    # -------------------------------------------------------------------- objs_hit

    def closest(self, O, D, lo, hi):
        """objs_hit (ray.fut:76-86) of rays (f64 origin, direction) with per-ray intervals (lo, hi): dict of t (-1 = no
        hit), leaf, sphere (caller's index), p, normal and margin."""
        m = len(O)
        lo = np.broadcast_to(np.asarray(lo, np.float64), (m,)).copy()
        hi = np.broadcast_to(np.asarray(hi, np.float64), (m,)).copy()
        P = self._pairs(O, D, np.minimum(lo, EPS), hi)
        ri, li, r1, r2, rs = P["ray"], P["leaf"], P["r1"], P["r2"], P["rs"]
        cand = np.where(r1 > EPS, r1, r2)
        ok = (P["disc"] > 0) & (cand > EPS) & (cand < hi[ri])
        g = self._reached(P, O, D, lo, hi)
        acc = ok & (g > 0)
        # winner: smallest t, then lowest leaf (the first one bvh_fold's left-first walk meets; closest_hit takes t < t_max)
        best_t = np.full(m, np.inf)
        best_leaf = np.full(m, -1, np.int64)
        k = np.nonzero(acc)[0]
        order = k[np.lexsort((li[k], cand[k], ri[k]))]
        first = order[np.unique(ri[order], return_index=True)[1]] if order.size else order
        best_t[ri[first]] = cand[first]
        best_leaf[ri[first]] = li[first]
        # margins of every pair that could have won, or could have taken the winner's place
        tw = best_t[ri]
        rel = cand <= np.where(np.isfinite(tw), tw * (1 + 1e-3) + 1e-9, np.inf)
        mg = np.minimum(P["dm"], self._rel(r1, EPS, rs))
        mg = np.where(r1 <= EPS * (1 + 1e-3), np.minimum(mg, self._rel(r2, EPS, rs)), mg)
        mg = np.minimum(mg, self._rel(cand, hi[ri], rs))
        mg = np.where(ok, np.minimum(mg, np.abs(g)), mg)
        other = acc & (best_leaf[ri] >= 0) & (self.geom[li] != self.geom[np.maximum(best_leaf[ri], 0)])
        mg = np.where(other, np.minimum(mg, self._rel(cand, tw, rs)), mg)
        margin = np.full(m, np.inf)
        np.minimum.at(margin, ri[rel], mg[rel])
        # the winner is intersected again on (t_min, t_best + 1) (ray.fut:85)
        hitm = best_leaf >= 0
        w = np.nonzero(hitm)[0]
        lw = best_leaf[w]
        oc = O[w] - self.C[lw]
        a, b = _dot(D[w], D[w]), _dot(oc, D[w])
        c = _dot(oc, oc) - self.rr[lw]
        disc = b * b - a * c
        sq = np.sqrt(np.maximum(disc, 0))
        q1, q2, qs = (-b - sq) / a, (-b + sq) / a, _root_scale(a, b, sq, _dot(oc, oc) + self.rr[lw])
        lo2 = np.full(len(w), EPS) if self.mutant == "reintersect_from_eps" else lo[w]
        hi2 = best_t[w] + 1.0
        in1 = (q1 > lo2) & (q1 < hi2)
        in2 = (q2 > lo2) & (q2 < hi2)
        t = np.where(in1, q1, np.where(in2, q2, -1.0))
        rm = np.minimum(self._rel(q1, lo2, qs), self._rel(q1, hi2, qs))
        rm = np.where(in1, rm, np.minimum(rm, np.minimum(self._rel(q2, lo2, qs), self._rel(q2, hi2, qs))))
        margin[w] = np.minimum(margin[w], rm)
        out_t = np.full(m, -1.0)
        out_leaf = np.full(m, -1, np.int64)
        out_t[w] = t
        out_leaf[w] = np.where(t >= 0, lw, -1)
        out_dm = np.ones(m)
        with np.errstate(invalid="ignore", divide="ignore"):
            out_dm[w] = np.abs(disc) / (b * b + np.abs(a * c))
        return self._records(O, D, out_t, out_leaf, margin, out_dm)

    def _records(self, O, D, t, leaf, margin, dm):
        """Hit records; `dm` is each hit's disc / (b^2 + |ac|): near grazing, a root's f32 error grows as
        1 / sqrt(dm) (comparisons widen their tolerance by it)."""
        hit = leaf >= 0
        lf = np.maximum(leaf, 0)
        p = np.where(hit[:, None], O + t[:, None] * D, 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            nrm = np.where(hit[:, None], (p - self.C[lf]) / self.rad[lf][:, None], 0.0)
        sphere = np.where(hit, lf if self.mutant == "no_perm" else self.perm[lf], -1)
        return dict(t=np.where(hit, t, -1.0), leaf=leaf, sphere=sphere, p=p, normal=nrm, margin=margin,
                    dm=np.where(hit, np.nan_to_num(dm, nan=1.0), 1.0))

    # -------------------------------------------------------------------- occlusion and multi-hit

    def _accepted(self, O, D, lo, hi):
        """The leaves bvh_fold reaches (boxes on (lo, hi)) whose sphere_hit L[i] r lo hi is a hit, without epsilon or
        re-intersection (include/ray_b200.h, occlusion and multi-hit): pairs with their t and margin."""
        P = self._pairs(O, D, lo, hi)
        ri, r1, r2, rs = P["ray"], P["r1"], P["r2"], P["rs"]
        l, h = lo[ri], hi[ri]
        in1 = (r1 > l) & (r1 < h)
        in2 = (r2 > l) & (r2 < h)
        ok = (P["disc"] > 0) & (in1 | in2)
        g = self._reached(P, O, D, lo, hi)
        mg = np.minimum(P["dm"], np.minimum(self._rel(r1, l, rs), self._rel(r1, h, rs)))
        mg = np.where(in1, mg, np.minimum(mg, np.minimum(self._rel(r2, l, rs), self._rel(r2, h, rs))))
        mg = np.where(ok, np.minimum(mg, np.abs(g)), mg)
        P.update(t=np.where(in1, r1, r2), acc=ok & (g > 0), mg=mg)
        return P

    @staticmethod
    def _intervals(m, lo, hi):
        lo = np.broadcast_to(np.asarray(lo, np.float64), (m,)).copy()
        hi = np.broadcast_to(np.asarray(hi, np.float64), (m,)).copy()
        bad = ~(np.isfinite(lo) & (lo >= 0) & np.isfinite(hi))      # the ranged queries' empty answer
        lo[bad], hi[bad] = 0.0, -1.0
        return lo, hi

    def occluded(self, O, D, lo, hi):
        """(occluded bool[m], margin[m]): a reached leaf's sphere is hit in (lo, hi).  The answer is robust when one
        accepted pair is, or else when every pair is robustly rejected."""
        m = len(O)
        lo, hi = self._intervals(m, lo, hi)
        P = self._accepted(O, D, lo, hi)
        ri = P["ray"]
        occ = np.zeros(m, bool)
        occ[ri[P["acc"]]] = True
        robust = np.zeros(m, bool)
        robust[ri[P["acc"] & (P["mg"] > TAU)]] = True
        margin = np.full(m, np.inf)
        np.minimum.at(margin, ri, P["mg"])
        return occ, np.where(robust, np.inf, margin)

    def multi_hits(self, O, D, lo, hi, k):
        """The k nearest accepted leaves by (t, leaf) and their count: (records dict of [m, k] arrays, count[m],
        margin[m]).  The count depends on every pair, so every pair's margin counts, and so do the gaps between the
        first k + 1 records of different geometry."""
        m = len(O)
        lo, hi = self._intervals(m, lo, hi)
        P = self._accepted(O, D, lo, hi)
        ri, li, t, rs = P["ray"], P["leaf"], P["t"], P["rs"]
        margin = np.full(m, np.inf)
        np.minimum.at(margin, ri, P["mg"])
        a = np.nonzero(P["acc"])[0]
        a = a[np.lexsort((li[a], t[a], ri[a]))]
        count = np.bincount(ri[a], minlength=m)
        start = np.concatenate([[0], np.cumsum(count)[:-1]])
        rank = np.arange(len(a)) - start[ri[a]]
        if len(a) > 1:   # consecutive records of one ray, different geometry, within the first k + 1
            same = (ri[a][1:] == ri[a][:-1]) & (rank[1:] <= k) & (self.geom[li[a][1:]] != self.geom[li[a][:-1]])
            gap = self._rel(t[a][1:], t[a][:-1], rs[a][1:])
            np.minimum.at(margin, ri[a][1:][same], gap[same])
        sel = a[rank < k]
        slot = rank[rank < k]
        tt = np.full((m, k), -1.0)
        leaf = np.full((m, k), -1, np.int64)
        dm = np.ones((m, k))
        tt[ri[sel], slot] = t[sel]
        leaf[ri[sel], slot] = li[sel]
        dm[ri[sel], slot] = P["dm"][sel]
        rec = self._records(np.repeat(O, k, 0), np.repeat(D, k, 0), tt.ravel(), leaf.ravel(), np.zeros(m * k), dm.ravel())
        rec = {key: v.reshape((m, k) + v.shape[1:]) for key, v in rec.items() if key != "margin"}
        return rec, count, margin

    # -------------------------------------------------------------------- ray_colour

    def _sky(self, D):
        """The sky colour of directions D (ray.fut:141-148)."""
        ud = _normalise(D)
        t = 0.5 * (ud[:, 0 if self.mutant == "sky_from_x" else 1] + 1.0)
        with np.errstate(invalid="ignore", over="ignore"):
            return (1.0 - t)[:, None] + t[:, None] * SKY

    def paths(self, O, D, max_depth=50):
        """ray_colour (ray.fut:126-148) in f64: (colour[m][3], segments[m], leaves[m][max_depth] (-1 after the last
        hit), margin[m]).  Every segment searches (0, 1e9)."""
        m = len(O)
        O, D = O.copy(), D.copy()
        light = np.ones((m, 3))
        colour = np.zeros((m, 3))
        seg = np.zeros(m, np.int64)
        leaves = np.full((m, max(max_depth, 1)), -1, np.int64)
        margin = np.full(m, np.inf)
        act = np.arange(m)
        depth = 0
        while act.size and depth < max_depth:
            h = self.closest(O[act], D[act], 0.0, 1e9)
            seg[act] += 1
            margin[act] = np.minimum(margin[act], h["margin"])
            hit = h["leaf"] >= 0
            leaves[act[hit], depth] = h["leaf"][hit]
            # miss: the sky (ray.fut:141-148)
            miss = act[~hit]
            with np.errstate(invalid="ignore", over="ignore"):
                colour[miss] = light[miss] * self._sky(D[miss])
            # hit: scatter (ray.fut:116-124)
            hh = act[hit]
            n = h["normal"][hit]
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                ud = _normalise(D[hh])
                refl = ud - (2.0 * _dot(ud, n))[:, None] * n
                dn = _dot(refl, n)
                margin[hh] = np.minimum(margin[hh], np.nan_to_num(np.abs(dn) / np.sqrt(_dot(refl, refl) * _dot(n, n)), nan=0.0))
                lc = self.col[h["leaf"][hit]]
                colour[hh] = light[hh] * colour[hh]
                on = dn > 0
                light[hh[on]] = light[hh[on]] * lc[on]
            O[hh[on]] = h["p"][hit][on]
            D[hh[on]] = refl[on]
            act = hh[on]
            depth += 1
        return colour, seg, leaves, margin

    def judged_paths(self, O, D, max_depth=50):
        """paths() plus the perturbation check.  The same path from the primary direction perturbed by PERTURB relative
        in two directions must give the same leaves; the colours' largest change is the sample's colour error estimate
        `err` (at least 1e-6), which must stay within COLOUR_TOL.  The f32 path's own error, from its hit points and
        normals as much as from its primary direction, stays within a few times err.  Returns (colour, seg,
        leaves, err, judged); err is relative to max(1, |c|)."""
        col, seg, leaves, margin = self.paths(O, D, max_depth)
        judged = margin > TAU
        err = np.full(len(O), 1e-6)
        for D2 in _perturbed(D):
            c2, s2, l2, _ = self.paths(O, D2, max_depth)
            with np.errstate(invalid="ignore"):
                dc = np.nan_to_num(np.abs(c2 - col) / np.maximum(1.0, np.abs(col)), nan=0.0).max(1)
            err = np.maximum(err, dc)
            judged &= (s2 == seg) & (l2 == leaves).all(1) & (np.isnan(c2) == np.isnan(col)).all(1)
        judged &= err <= COLOUR_TOL
        return col, seg, leaves, err, judged

    def pixels(self, h, w, j, i, spp, cam7=None, max_depth=50):
        """Pixels (row j, column i) of an h x w frame at spp: (packed int32, float colour = mean of the samples, err,
        judged): a pixel is judged if all its samples are and its mean is QUANT_TAU plus its error estimate from a
        quantisation step."""
        cam7 = self.cam7 if cam7 is None else cam7
        j, i = np.asarray(j), np.asarray(i)
        jj, ii, ss = np.repeat(j, spp), np.repeat(i, spp), np.tile(np.arange(spp), len(j))
        O, D = primary_rays(cam7, h, w, jj, ii, ss, self.mutant)
        col, _, _, err, judged = self.judged_paths(O, D, max_depth)
        mean = col.reshape(len(j), spp, 3).mean(1)
        err = err.reshape(len(j), spp).max(1)
        pix, qm = quantise(mean)
        scale = np.nan_to_num(np.maximum(1.0, np.abs(mean)).max(1), nan=1.0, posinf=1.0)
        return pix, mean, err, judged.reshape(len(j), spp).all(1) & (qm > QUANT_TAU + 255.99 * err * scale)

    def samples(self, h, w, j, i, s, cam7=None, max_depth=50):
        """Sample s of pixel (row j, column i) of an h x w frame, for integer arrays j, i, s (broadcast together):
        (colour [..., 3], err [...], judged [...]) of judged_paths.  Samples of one pixel whose offsets coincide (every
        sample from 2^23 / c on is the sample-0 ray, and the offsets are quarters or halves from 2^21 / c on) are one
        ray, traced once."""
        cam7 = self.cam7 if cam7 is None else cam7
        j, i, s = np.broadcast_arrays(np.asarray(j, np.int64), np.asarray(i, np.int64), np.asarray(s, np.int64))
        ox, oy = sample_offsets(s.ravel(), self.mutant)
        key = np.stack([j.ravel().astype(np.float64), i.ravel().astype(np.float64), ox, oy], 1)
        uniq, inv = np.unique(key, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        O, D = offset_rays(cam7, h, w, uniq[:, 0], uniq[:, 1], uniq[:, 2], uniq[:, 3], self.mutant)
        col, _, _, err, judged = self.judged_paths(O, D, max_depth)
        return col[inv].reshape(s.shape + (3,)), err[inv].reshape(s.shape), judged[inv].reshape(s.shape)

    # -------------------------------------------------------------------- G-buffer

    def gbuffer(self, h, w, j, i, spp, cam7=None):
        """The first-hit buffers of pixels (row j, column i) of an h x w frame at spp (include/ray_b200.h,
        ray_b200_render_gbuffer), from closest(ray, 0, 1e9) of every sample's camera ray: id, the caller's index of
        sample 0's sphere (-1 on a miss); depth, sample 0's t (-1); coverage, how many samples hit; normal and albedo,
        means over the samples of the hit normal (0 on a miss) and of the hit sphere's colour (the sky colour of the
        ray on a miss).  Returns (buffers dict, judged [n], records): a pixel is judged when every sample's margin
        exceeds TAU and both perturbed directions of every sample hit the same sphere; records are closest()'s of
        every sample, shaped [n, spp, ...], with the rays' origins and directions under "O" and "D"."""
        cam7 = self.cam7 if cam7 is None else cam7
        j, i = np.asarray(j), np.asarray(i)
        n = len(j)
        O, D = primary_rays(cam7, h, w, np.repeat(j, spp), np.repeat(i, spp), np.tile(np.arange(spp), n), self.mutant)
        rec = self.closest(O, D, 0.0, 1e9)
        judged = rec["margin"] > TAU
        for D2 in _perturbed(D):
            judged &= self.closest(O, D2, 0.0, 1e9)["leaf"] == rec["leaf"]
        hit = rec["leaf"] >= 0
        sky = np.zeros((len(O), 3)) if self.mutant == "gbuffer_miss_albedo_black" else self._sky(D)
        albedo = np.where(hit[:, None], self.col[np.maximum(rec["leaf"], 0)], sky)
        rec = {k: v.reshape((n, spp) + v.shape[1:]) for k, v in dict(rec, O=O, D=D).items()}
        first = -1 if self.mutant == "gbuffer_depth_last_sample" else 0
        ident = np.where(rec["leaf"][:, 0] >= 0, rec["leaf"][:, 0], -1) if self.mutant == "gbuffer_id_in_leaf_order" \
            else rec["sphere"][:, 0]
        out = dict(id=ident, depth=rec["t"][:, first], coverage=hit.reshape(n, spp).sum(1),
                   normal=rec["normal"].mean(1), albedo=albedo.reshape(n, spp, 3).mean(1))
        return out, judged.reshape(n, spp).all(1), rec

    # -------------------------------------------------------------------- the noise estimate

    def m2(self, colours):
        """(sum, M2) of colours float64 [..., n, 3] over their samples (axis -2), by Welford's update in f64: M2 += (x_k -
        S_k / k) (x_k - S_{k+1} / (k + 1)) after sample k >= 1, which is the sum of squared deviations from the mean, so
        M2 / (n - 1) is the unbiased sample variance (include/ray_b200.h, ray_b200_render_adaptive_var)."""
        x = np.asarray(colours, np.float64)
        S, M = x[..., 0, :].copy(), np.zeros_like(x[..., 0, :])
        with np.errstate(invalid="ignore", over="ignore"):
            for k in range(1, x.shape[-2]):
                xk = x[..., k, :]
                nxt = S + xk
                if self.mutant == "welford_old_mean":
                    M = M + (xk - S / k) ** 2
                else:
                    M = M + (xk - S / k) * (xk - nxt / (k + 1))
                S = nxt
        return S, M

    def select(self, S, M2, n, rel_err, mean_floor, min_count, max_count):
        """ray_b200_adaptive_select in f64 on sums S [..., 3] and M2 [..., 3] of n samples (n [...] int): (mask, E, T)
        where E = sum of M2 / (n (n - 1)), the variance of the mean summed over the channels, T = (rel_err (sum of S / n
        + mean_floor))^2, and the mask is 0 <= n < max_count and (n < min_count or E > T)."""
        n = np.asarray(n, np.float64)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            v = np.asarray(M2, np.float64).sum(-1)
            E = v / (n - 1) if self.mutant == "select_without_count" else v / (n * (n - 1))
            T = (rel_err * (np.asarray(S, np.float64).sum(-1) / n + mean_floor)) ** 2
            mask = (n >= 0) & (n < max_count) & ((n < min_count) | (E > T))
        return mask, E, T


def m2_bound(x, delta):
    """A bound on |M2_f32 - M2| per channel, where M2 is the f64 sum of squared deviations of the f64 colours x
    [..., n, 3] and M2_f32 is Welford's update run in f32 on colours within delta [..., n, 3] of x:

    * the propagated colour error: moving each x_k by at most D = max delta moves each deviation x_k - mean by at most
      2 D, so M2 moves by at most 4 D sum|x_k - mean| + 4 n D^2;
    * Welford's f32 error: the running sum S_k is within (k - 1) k u X of its exact value (u = 2^-24, X = max |x_k|), so
      S_k / k is within (k + 1) u X, each factor x_k - S_k / k within (k + 3) u X and each term within 4 (k + 4) u X^2;
      over n - 1 terms that is 2 (n + 4)^2 u X^2, and the n - 1 additions of the terms add (n - 1) u M2.

    Twice that sum is returned.  Everything here is finite; NaN colours are compared as NaN."""
    x = np.asarray(x, np.float64)
    n = x.shape[-2]
    D = np.asarray(delta, np.float64).max(-2)
    X = np.abs(x).max(-2) + D
    dev = np.abs(x - x.mean(-2, keepdims=True)).sum(-2)
    M2 = ((x - x.mean(-2, keepdims=True)) ** 2).sum(-2)
    return 2 * (4 * D * dev + 4 * n * D * D + 2 * (n + 4) ** 2 * U32 * X * X + (n - 1) * U32 * (M2 + 4 * D * dev))
