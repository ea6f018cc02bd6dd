"""Scene and ray constructors for tests/test_limits.py: scenes that sit at the limits prepare_scene, render and the ray
queries accept (deepest trees, 2^26 spheres, exact ties, paths that bounce for a chosen number of segments), and the
numpy helpers that check their premises from a dumped tree.  TEST INFRASTRUCTURE ONLY.

Every scene here puts its sphere centres on integers inside [0, 1024]^3 with the centre box exactly [0, 1024]^3, so a
centre's Morton key (bvh.fut:15-41) is known in advance: the normalised coordinate c / 1024 times 1024 is c again, and
each axis contributes floor(min(c, 1023)).
"""
import numpy as np

import ray_query_oracle as Q

# ------------------------------------------------------------------------------------------ Morton keys


def expand_bits(v):
    v = np.asarray(v, np.uint64)
    v = (v * 0x00010001) & 0xFF0000FF
    v = (v * 0x00000101) & 0x0F00F00F
    v = (v * 0x00000011) & 0xC30C30C3
    v = (v * 0x00000005) & 0x49249249
    return v.astype(np.uint32)


def morton_of_cell(x, y, z):
    """Key of a centre whose quantised cell is (x, y, z), each in [0, 1023] (bit 3k+2 = x bit k, 3k+1 = y, 3k = z)."""
    return (expand_bits(x) * np.uint32(4) + expand_bits(y) * np.uint32(2) + expand_bits(z)).astype(np.uint32)


# ------------------------------------------------------------------------------------------ deepest trees

COMB_LEVELS = 30   # one comb level per bit of the 30-bit Morton key


def comb_scene(m, cluster_radius=1.0):
    """The deepest tree a scene of about m spheres can have.

    m coincident spheres at the origin (key 0, distinct colours) sit under a comb over the 30 Morton key bits: for key bit
    b there is a PAIR of spheres whose key is exactly 1 << b, so the pair is an inner node of its own (split by index) and
    every comb node has two inner children.  The root splits at bit 29, its left child at bit 28, ... and the node of bit 0
    has the cluster as its left child, so the cluster's subtree starts at depth 30 and its leaves, split purely by index,
    are at depth 30 + ceil(log2 m).  A corner sphere at (1024, 1024, 1024) fixes the centre box (its key is 0x3fffffff).

    The comb spheres have radii larger than their distance to the origin: their boxes, and every refitted box of the comb,
    cover the cluster, so a ray through the cluster's box passes the box tests at every level and defers a sibling at each.
    Returns (spheres float32[61 + m][7], index of the first cluster sphere in the array)."""
    rows = []
    for b in range(COMB_LEVELS):
        axis, k = 2 - b % 3, b // 3        # bit 3k+2 -> x, 3k+1 -> y, 3k -> z
        c = [0.0, 0.0, 0.0]
        c[axis] = float(1 << k)
        for extra in (4.0, 5.0):           # radius > distance to the origin + the cluster's extent
            rows.append([*c, 0.2 + 0.02 * b, 0.5, 0.9 - 0.02 * b, float(1 << k) + extra])
    rows.append([1024.0, 1024.0, 1024.0, 0.9, 0.9, 0.9, 1.0])
    head = np.array(rows, np.float32)
    cl = np.zeros((m, 7), np.float32)
    i = np.arange(m, dtype=np.float32)
    cl[:, 3] = 0.25 + 0.5 * ((i % 7) / 6)
    cl[:, 4] = 0.25 + 0.5 * ((i % 11) / 10)
    cl[:, 5] = 0.25 + 0.5 * ((i % 13) / 12)
    cl[:, 6] = cluster_radius
    return np.ascontiguousarray(np.concatenate([head, cl]), np.float32), head.shape[0]


# camera outside every comb sphere, looking at the cluster; with a 3-degree field of view a few dozen pixels of a 48 x 64
# frame see the cluster's box, so the oracle's frame stays cheap although each of them tests all m cluster leaves
COMB_CAM = np.float32([-300, -290, -310, 0, 0, 0, 3])


def comb_query_rays(n_random, seed):
    """Rays that start inside every comb sphere, 3 units from the origin, and aim at the cluster (radius 1): the first
    six along the axes with exactly representable hits (t = 2, p = -d, normal = -d), then n_random with random origins on
    the radius-3 sphere aimed at random points of the cluster's inner half."""
    axes = np.float32([[1, 0, 0], [0, 1, 0], [0, 0, 1], [-1, 0, 0], [0, -1, 0], [0, 0, -1]])
    exact = np.concatenate([-3 * axes, axes], 1)
    rng = np.random.default_rng(seed)
    o = rng.standard_normal((n_random, 3))
    o = 3.0 * o / np.linalg.norm(o, axis=1, keepdims=True)
    target = rng.uniform(-0.5, 0.5, (n_random, 3))
    d = target - o
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    return np.ascontiguousarray(np.concatenate([exact, np.concatenate([o, d], 1).astype(np.float32)]), np.float32)


def leaf_depths(tree):
    """Depth (root = 0) of every inner node and every leaf of a dumped tree (left/right: inner i -> i, leaf i -> ~i)."""
    left, right = np.asarray(tree["left"]), np.asarray(tree["right"])
    ni = left.shape[0]
    inner = np.full(ni, -1, np.int64)
    leaf = np.full(ni + 1, -1, np.int64)
    frontier, d = np.array([0]), 0
    while frontier.size:
        inner[frontier] = d
        nxt = []
        for ch in (left[frontier], right[frontier]):
            leaf[~ch[ch < 0]] = d + 1
            nxt.append(ch[ch >= 0])
        frontier, d = np.concatenate(nxt), d + 1
    assert (inner >= 0).all() and (leaf >= 0).all(), "the tree is not connected"
    return inner, leaf


def _slab_hit(box, o, d, shrink):
    """float64 slab test of the ray's whole line (t in (0, inf)) against box shrunk by `shrink` on every side."""
    lo = np.asarray(box[:3], np.float64) + shrink
    hi = np.asarray(box[3:], np.float64) - shrink
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / np.asarray(d, np.float64)
        t0 = (lo - o) * inv
        t1 = (hi - o) * inv
    tmin = np.nanmax(np.concatenate([np.minimum(t0, t1), [0.0]]))
    tmax = np.nanmin(np.maximum(t0, t1))
    return tmax > tmin


def deferred_siblings(tree, spheres, ray, leaf, shrink=1e-3):
    """Number of inner nodes on the path root -> `leaf` (a sorted leaf index) whose BOTH children's boxes the ray passes,
    each tested in float64 against the box shrunk by `shrink`: a stack walk reaching that leaf holds at least this many
    deferred siblings (the boxes are the reference's refitted ones; a leaf's box is its sphere's)."""
    left, right, parent = tree["left"], tree["right"], tree["parent"]
    boxes, perm = tree["boxes"], tree["perm"]
    o, d = np.asarray(ray[:3], np.float64), np.asarray(ray[3:], np.float64)

    def box_of(child):
        if child >= 0:
            return boxes[child]
        s = spheres[perm[~child]]
        return np.concatenate([s[:3] - s[6], s[:3] + s[6]])

    node = int(np.nonzero(left == ~leaf)[0][0]) if (left == ~leaf).any() else int(np.nonzero(right == ~leaf)[0][0])
    count = 0
    while node >= 0:
        if _slab_hit(box_of(left[node]), o, d, shrink) and _slab_hit(box_of(right[node]), o, d, shrink):
            count += 1
        node = int(parent[node])
    return count


# ------------------------------------------------------------------------------------------ 2^26 spheres

TOP_TARGETS = 32


def top_of_index_scene(n):
    """n spheres whose last TOP_TARGETS in Morton order are targets with exactly representable answers.

    n - 32 filler spheres (radius 0.25) on the integer grid [0, 512) x [0, 512) x [0, 256) - every cell key below 7 << 27 -
    and 32 targets (radius 1) at (1024 - 8 j, 1024, 1024), whose keys are above every filler key and increase with x.
    Target j sits at caller index targets[j] and at sorted leaf n - 1 - j.  Returns (spheres, cam7, targets)."""
    nf = n - TOP_TARGETS
    s = np.empty((n, 7), np.float32)
    targets = (np.arange(TOP_TARGETS, dtype=np.int64) * (n // TOP_TARGETS) + 12345) % n
    is_target = np.zeros(n, bool)
    is_target[targets] = True
    fill = np.nonzero(~is_target)[0]
    g = np.arange(nf, dtype=np.int64)
    s[fill, 0] = (g & 511).astype(np.float32)
    s[fill, 1] = ((g >> 9) & 511).astype(np.float32)
    s[fill, 2] = (g >> 18).astype(np.float32)
    s[fill, 3] = 0.3 + 0.6 * (g & 15).astype(np.float32) / 15
    s[fill, 4] = 0.3 + 0.6 * ((g >> 4) & 15).astype(np.float32) / 15
    s[fill, 5] = 0.6
    s[fill, 6] = 0.25
    j = np.arange(TOP_TARGETS)
    s[targets, 0] = (1024 - 8 * j).astype(np.float32)
    s[targets, 1] = 1024
    s[targets, 2] = 1024
    s[targets, 3] = (1 + j).astype(np.float32) / 40
    s[targets, 4] = 0.5
    s[targets, 5] = 0.75
    s[targets, 6] = 1
    assert nf <= 512 * 512 * 256
    cam = np.float32([900, 1100, 1100, 900, 1024, 1024, 40])
    return s, cam, targets


def top_target_cases():
    """(ray, t, p, normal) of target j: straight down onto its top, t = 9, p = centre + (0, 0, 1), normal (0, 0, 1)."""
    out = []
    for j in range(TOP_TARGETS):
        x = np.float32(1024 - 8 * j)
        out.append(([x, 1024, 1034, 0, 0, -1], 9.0, [x, 1024, 1025], [0, 0, 1]))
    return out


# ------------------------------------------------------------------------------------------ frame rows


def camera_rays_rows(camera, h, w, rows):
    """The camera rays of whole rows `rows` of an h x w frame at 1 spp, float32[len(rows)][w][6], with the operations of
    raytracers_b200.camera_rays (which the suite checks against the oracle's get_ray) but without the full frame."""
    c = np.asarray(camera, np.float32).reshape(12)
    f = np.float32
    i = np.arange(w, dtype=np.float32)[None, :]
    hj = (f(h) - np.asarray(rows, np.int64).astype(np.float32))[:, None]
    u = np.broadcast_to(i / f(w), (len(rows), w))
    v = np.broadcast_to(hj / f(h), (len(rows), w))
    out = np.empty((len(rows), w, 6), np.float32)
    out[..., 0:3] = c[0:3]
    for a in range(3):
        out[..., 3 + a] = ((c[3 + a] + u * c[6 + a]) + v * c[9 + a]) - c[a]
    return out


# ------------------------------------------------------------------------------------------ paths that bounce k times

FACING_CAM = np.float32([30, 0, 0, 0, 0, 0, 60])


def facing_spheres(radius, gap):
    """Two white spheres on the z axis whose facing poles are `gap` apart around the origin: a ray on the axis bounces
    between them forever (every hit point, normal and reflection is exact); a ray offset from the axis by e leaves after
    a number of bounces that grows as e shrinks (both mirrors are convex)."""
    r = np.float32(radius)
    z = np.float32(radius + gap / 2)
    return np.array([[0, 0, -z, 1, 1, 1, r], [0, 0, z, 1, 1, 1, r]], np.float32)


def axis_ray(offset):
    return [np.float32(offset), 0, 0, 0, 0, 1]


def bounce_count(pr, offset, limit=65535):
    """Objs_hit calls of the oracle's path from axis_ray(offset) with depth limit `limit`, and whether it escaped."""
    rgb, seg = pr.trace_paths(np.array([axis_ray(offset)], np.float32), max_depth=limit)
    return int(seg[0]), bool(rgb[0].any())


def rays_escaping_after(pr, segments, lo_exp, hi_exp, steps=4096):
    """For each wanted segment count k, one offset along the axis whose oracle path escapes to the sky in exactly k
    segments (k - 1 bounces).  Scans offsets 2^-x for x in [lo_exp, hi_exp] and bisects between neighbours.  Returns
    {k: offset}; counts the scan cannot produce are missing."""
    xs = np.linspace(lo_exp, hi_exp, steps)
    offs = (2.0 ** -xs).astype(np.float32)
    rays = np.zeros((steps, 6), np.float32)
    rays[:, 0] = offs
    rays[:, 5] = 1
    rgb, seg = pr.trace_paths(rays, max_depth=65535)
    esc = rgb.any(1)
    found = {}
    for k in segments:
        hit = np.nonzero(esc & (seg == k))[0]
        if hit.size:
            found[k] = float(offs[hit[0]])
            continue
        # bisect between the last offset below k and the first above (offsets shrink as x grows: segments grow)
        below = np.nonzero(esc & (seg < k))[0]
        above = np.nonzero(esc & (seg > k))[0]
        if not below.size or not above.size:
            continue
        a, b = offs[below[-1]], offs[above[above > below[-1]][0]] if (above > below[-1]).any() else None
        if b is None:
            continue
        for _ in range(64):
            mid = np.float32(np.sqrt(np.float64(a) * np.float64(b)))
            if mid == a or mid == b:
                break
            s, e = bounce_count(pr, mid)
            if e and s == k:
                found[k] = float(mid)
                break
            if e and s < k:
                a = mid
            else:
                b = mid
    return found


# ------------------------------------------------------------------------------------------ exact ties

TIE_SIZES = (2, 3, 31, 32, 33, 100)


def tie_groups(sizes=TIE_SIZES, seed=5, filler=0):
    """Groups of coincident copies (radius 16, distinct colours) at (64 + 40 g, 512, 512), one per size, their copies
    scattered through the caller's array in random order; optionally `filler` small random spheres elsewhere in the
    centre box, so that a tree of the scene is larger than the staging area.  Corner spheres at (0,0,0) and
    (1024,1024,1024) fix the centre box.  Returns (spheres, groups: list of int arrays of caller indices)."""
    rng = np.random.default_rng(seed)
    rows, gid = [], []
    for g, size in enumerate(sizes):
        for c in range(size):
            col = rng.uniform(0.2, 1.0, 3)
            rows.append([64 + 40 * g, 512, 512, *col, 16.0])
            gid.append(g)
    for p in ((0, 0, 0), (1024, 1024, 1024)):
        rows.append([*p, 0.5, 0.5, 0.5, 1.0])
        gid.append(-1)
    if filler:
        f = np.empty((filler, 7))
        f[:, 0] = rng.uniform(0, 1024, filler)
        f[:, 1] = rng.uniform(0, 400, filler)   # below the groups' row: the frames look at the groups from above
        f[:, 2] = rng.uniform(0, 1024, filler)
        f[:, 3:6] = rng.uniform(0.2, 1.0, (filler, 3))
        f[:, 6] = rng.uniform(0.5, 3.0, filler)
        rows.extend(f.tolist())
        gid.extend([-1] * filler)
    order = rng.permutation(len(rows))
    s = np.array(rows, np.float32)[order]
    gid = np.array(gid)[order]
    return np.ascontiguousarray(s), [np.sort(np.nonzero(gid == g)[0]) for g in range(len(sizes))]


TIE_CAM = np.float32([164, 690, 600, 164, 512, 512, 75])


def tie_rays(groups_count):
    """Per group: rays along +z, -z, +x and -y onto its centre from 20 units away (t = 4 at radius 16, p = the pole,
    normal = -direction), and one ray along +z offset by (0.5, 0.25) (inexact, compared with the oracle only)."""
    rays = []
    for g in range(groups_count):
        c = np.float32([64 + 40 * g, 512, 512])
        for d in ([0, 0, 1], [0, 0, -1], [1, 0, 0], [0, -1, 0]):
            d = np.float32(d)
            rays.append([*(c - 20 * d), *d])
        rays.append([c[0] + 0.5, c[1] + 0.25, c[2] - 20, 0, 0, 1])
    return np.array(rays, np.float32)


def prepare_oracle(spheres, cam, h, w):
    return Q.prepare_custom(spheres, cam, h, w)
