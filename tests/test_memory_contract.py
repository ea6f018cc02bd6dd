"""Memory the library must not touch, scratch it must not trust, and schedules it must not depend on.

The other GPU tests ask whether an answer is the oracle's.  Three kinds of bug pass that question unchanged, and this file
asks about them:

- Writes outside the contract.  Every output of every entry point that writes device memory is a guarded buffer,
  guard | payload | guard with 4 KiB guards, filled with a sentinel byte.  After the call every guard byte still holds the
  sentinel, every element the contract defines equals the oracle (or the rule the call's own test file states), and every
  element the contract says is neither read nor written (unselected adaptive pixels, other ranks' pixels of a shard's
  row-major frame) still holds the sentinel.  Each case runs with the sentinels 0x00 and 0xFF (a NaN in every float, -1
  in every int), and the defined elements must be bit-identical across the two.  Caller inputs (rays, camera tables,
  sphere records, masks, the sums and counts of unselected pixels) come back unchanged byte for byte.
- Reads of memory nobody wrote.  Before every library call the device's default stream-ordered pool, from which the
  library takes its scratch, is filled with a pattern through the driver API (libcuda.so.1 with ctypes), on the stream
  the context launches on, where stream-ordered reuse is guaranteed.  The context's grow-only cudaMalloc scratch is
  dropped first (futhark_context_clear_caches) and a block of the driver's plain allocator is filled with the pattern
  too.  A premise check reads the pattern back from allocations of the test's own.  Every output must be bit-identical
  across the patterns 0x00, 0xFF and 0x7F and equal to the oracle.
- Schedule dependence.  The warp-queue kernel is persistent and claims work through global counters and shared-memory
  queues; its answers must not depend on how the hardware schedules its warps.  Frames and queries run from two host
  threads on two contexts at once, next to a matmul workload that holds SMs, and on smaller grids and other claim orders
  (wq_warps, permute, heavy_first, probe_segments), all bit for bit against the oracle.

Limits.  The pool can only be poisoned where it has free memory: memory freed into a chunk that a prepared scene still
uses is poisoned by the small blocks of the fill when the pool hands them out there, which the driver does not promise.
Reuse of a block freed with cuMemFree by the library's next cudaMalloc is not guaranteed either, and the premise check
covers the pool only: on an H100 a cuMemAlloc right after the fill returned the pattern for the 1 MiB block and fresh
memory for the 8, 64 and 256 MiB ones, so of the grow-only scratch only blocks of about a MiB are likely to be poisoned.
"""
import ctypes as C
import functools
import itertools
import threading

import numpy as np
import pytest

import limit_scenes as LS
import ray_query_oracle as Q      # tests/ray_query_oracle.py: the CPU oracle of the ray queries
import raytracers_b200 as RB
from oracle import pyoracle as O
from ray_query_cases import bits_differ, hits_differ, quantise, random_rays
from raytracers_b200 import distributed as D
from test_render_accumulate import frame_of, sequential_sum
from test_render_adaptive import ragged_model, random_masks
from test_render_adaptive_var import m2_model, select_model
from test_render_gbuffer import OUTPUTS as GB_OUTPUTS, gbuffer_rule
from test_render_views import poses

GUARD = 4096
SENTINELS = (0x00, 0xFF)
PATTERNS = (0x00, 0xFF, 0x7F)
SHAPES = [(1, 1), (1, 37), (37, 1), (3, 5), (8, 4), (9, 5), (33, 65)]
SCENE_NAMES = ("rgbbox", "irreg", "comb")
RAY_COUNTS = [1, 31, 32, 33, 1000]
KS = [1, 7, 64]
WORLD = 3
K_MAX_DEPTH = 50          # render_params.h kMaxDepth: the longest path, and the most probe segments a tile can take

# ------------------------------------------------------------------------------------------ guarded buffers


def _torch():
    import torch
    return torch


class Guarded:
    """A uint8 torch buffer laid out as guard | payload | guard, every byte filled with `sentinel`, or the payload with
    the bytes of `data` (an input).  `ptr` is the payload's address: 16-byte aligned, or with align=4 exactly 4 bytes
    past a 16-byte boundary (for the buffers the header allows to be 4-byte aligned)."""

    def __init__(self, nbytes, sentinel, align=16, guard=GUARD, device="cuda", data=None):
        if not isinstance(sentinel, int) or not 0 <= sentinel <= 255:
            raise ValueError(f"sentinel must be a byte, got {sentinel!r}")
        if align not in (4, 16):
            raise ValueError(f"align must be 4 or 16, got {align!r}")
        if guard < GUARD or guard % 16:
            raise ValueError(f"guard must be a multiple of 16 of at least {GUARD} bytes, got {guard!r}")
        if data is not None:
            data = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
            nbytes = data.size
        if int(nbytes) < 0:
            raise ValueError(f"nbytes must be >= 0, got {nbytes}")
        torch = _torch()
        self.sentinel, self.nbytes, self.offset = sentinel, int(nbytes), guard + (0 if align == 16 else 4)
        self.buf = torch.full((self.offset + self.nbytes + guard,), sentinel, dtype=torch.uint8, device=device)
        if data is not None:
            self.buf[self.offset:self.offset + self.nbytes].copy_(torch.from_numpy(data.copy()))
        self.ptr = self.buf.data_ptr() + self.offset
        assert self.ptr % 16 == self.offset % 16, "torch's allocation is not 16-byte aligned"

    def check(self, what):
        """Asserts that every guard byte still holds the sentinel; returns the payload's bytes (numpy uint8)."""
        host = self.buf.cpu().numpy()
        lead, body, trail = host[:self.offset], host[self.offset:self.offset + self.nbytes], host[self.offset + self.nbytes:]
        bad_lead, bad_trail = np.flatnonzero(lead != self.sentinel), np.flatnonzero(trail != self.sentinel)
        assert bad_lead.size == 0, f"{what}: {bad_lead.size} bytes written before the buffer (first at {bad_lead[-1] - lead.size})"
        assert bad_trail.size == 0, f"{what}: {bad_trail.size} bytes written past the end of the buffer (first at +{bad_trail[0]})"
        return body.copy()


def run_call(e, call, outs, ins=None, sentinel=0, what=""):
    """One library call on guarded buffers.  outs: {name: nbytes | initial contents (an in-out buffer)}; ins: {name:
    (array, align)}, read-only inputs.  call(ptrs) makes the call.  Checks every guard and every input, and returns
    {name: payload bytes} of the outputs."""
    torch = _torch()
    ins = ins or {}
    ob = {k: Guarded(v, sentinel) if isinstance(v, (int, np.integer)) else Guarded(0, sentinel, data=v) for k, v in outs.items()}
    ib = {k: Guarded(0, sentinel, align=a, data=arr) for k, (arr, a) in ins.items()}
    torch.cuda.current_stream().synchronize()   # the fills ran on torch's stream; the context launches on its own
    e.before_call()
    call({**{k: b.ptr for k, b in ob.items()}, **{k: b.ptr for k, b in ib.items()}})
    e.ctx.sync()
    for k, b in ib.items():
        got = b.check(f"{what} input {k}")
        assert np.array_equal(got, np.ascontiguousarray(ins[k][0]).view(np.uint8).reshape(-1)), f"{what}: input {k} was written"
    return {k: b.check(f"{what} {k}") for k, b in ob.items()}


def as_(payload, dtype, shape):
    return payload.view(dtype).reshape(shape)


def assert_bits(got, want, what):
    bad = bits_differ(got, want)
    assert bad == 0, f"{what}: {bad} values differ"


def assert_equal(got, want, what):
    bad = int((np.asarray(got) != np.asarray(want)).sum())
    assert bad == 0, f"{what}: {bad} of {np.asarray(want).size} values differ"


def assert_untouched(payload, per_elem, keep, sentinel, what):
    """payload bytes of an output of elements of per_elem bytes: the elements where keep is True hold the sentinel."""
    el = payload.reshape(-1, per_elem)[np.asarray(keep).reshape(-1)]
    assert (el == sentinel).all(), f"{what}: {int((el != sentinel).any(1).sum())} elements outside the contract were written"


# ------------------------------------------------------------------------------------------ the driver's allocators

_POOL_FILL = [512 << 20] + [4 << 20] * 16 + [256 << 10] * 64 + [16 << 10] * 128 + [512] * 256
_PLAIN_FILL = [256 << 20, 64 << 20, 8 << 20, 1 << 20]
_PREMISE = [512, 16 << 10, 256 << 10, 4 << 20]


def poison_args(pattern, sizes):
    """(pattern, sizes) checked: a byte, and a non-empty list of positive block sizes."""
    if isinstance(pattern, bool) or not isinstance(pattern, (int, np.integer)) or not 0 <= int(pattern) <= 255:
        raise ValueError(f"pattern must be a byte (0..255), got {pattern!r}")
    sizes = [int(s) for s in sizes]
    if not sizes or any(s <= 0 for s in sizes):
        raise ValueError(f"block sizes must be positive, got {sizes}")
    return int(pattern), sizes


class Driver:
    """The CUDA driver API (libcuda.so.1) through ctypes, for the pool and plain allocations of the poisoning."""

    def __init__(self, device=0):
        L = C.CDLL("libcuda.so.1")
        vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
        sig = {"cuDeviceGet": [C.POINTER(C.c_int), C.c_int], "cuDeviceGetDefaultMemPool": [C.POINTER(vp), C.c_int],
               "cuMemAllocFromPoolAsync": [C.POINTER(u64), sz, vp, vp], "cuMemsetD8Async": [u64, C.c_ubyte, sz, vp],
               "cuMemFreeAsync": [u64, vp], "cuMemAlloc_v2": [C.POINTER(u64), sz], "cuMemsetD8_v2": [u64, C.c_ubyte, sz],
               "cuMemFree_v2": [u64], "cuStreamSynchronize": [vp], "cuMemcpyDtoH_v2": [vp, u64, sz]}
        for name, args in sig.items():
            getattr(L, name).argtypes = args
            getattr(L, name).restype = C.c_int
        self.L = L
        dev = C.c_int(0)
        self._ok(L.cuDeviceGet(C.byref(dev), int(device)), "cuDeviceGet")
        pool = C.c_void_p(None)
        self._ok(L.cuDeviceGetDefaultMemPool(C.byref(pool), dev), "cuDeviceGetDefaultMemPool")
        self.pool = pool

    @staticmethod
    def _ok(rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed with CUresult {rc}")

    def poison_pool(self, stream, pattern, sizes=_POOL_FILL):
        """Allocates blocks of `sizes` from the default pool on `stream`, fills them with `pattern` and frees them on
        the same stream, so that the pool's next allocations on that stream return the pattern."""
        pattern, sizes = poison_args(pattern, sizes)
        L, s, ptrs = self.L, C.c_void_p(int(stream)), []
        for n in sizes:
            p = C.c_uint64(0)
            self._ok(L.cuMemAllocFromPoolAsync(C.byref(p), n, self.pool, s), "cuMemAllocFromPoolAsync")
            self._ok(L.cuMemsetD8Async(p, pattern, n, s), "cuMemsetD8Async")
            ptrs.append(p)
        for p in ptrs:
            self._ok(L.cuMemFreeAsync(p, s), "cuMemFreeAsync")
        self._ok(L.cuStreamSynchronize(s), "cuStreamSynchronize")

    def poison_plain(self, pattern, sizes=_PLAIN_FILL):
        """cuMemAlloc / cuMemsetD8 / cuMemFree of blocks of `sizes`: what cudaMalloc returns next likely holds the
        pattern (the driver does not promise it)."""
        pattern, sizes = poison_args(pattern, sizes)
        ptrs = []
        for n in sizes:
            p = C.c_uint64(0)
            self._ok(self.L.cuMemAlloc_v2(C.byref(p), n), "cuMemAlloc")
            self._ok(self.L.cuMemsetD8_v2(p, pattern, n), "cuMemsetD8")
            ptrs.append(p)
        for p in ptrs:
            self._ok(self.L.cuMemFree_v2(p), "cuMemFree")

    def pool_reads_back(self, stream, pattern, sizes=_PREMISE):
        """Premise of the poisoning: allocations from the pool on `stream` hold the pattern.  Frees them again."""
        pattern, sizes = poison_args(pattern, sizes)
        L, s, ok = self.L, C.c_void_p(int(stream)), True
        for n in sizes:
            p = C.c_uint64(0)
            self._ok(L.cuMemAllocFromPoolAsync(C.byref(p), n, self.pool, s), "cuMemAllocFromPoolAsync")
            self._ok(L.cuStreamSynchronize(s), "cuStreamSynchronize")
            host = np.empty(n, np.uint8)
            self._ok(L.cuMemcpyDtoH_v2(host.ctypes.data_as(C.c_void_p), p, n), "cuMemcpyDtoH")
            ok &= bool((host == pattern).all())
            self._ok(L.cuMemFreeAsync(p, s), "cuMemFreeAsync")
        self._ok(L.cuStreamSynchronize(s), "cuStreamSynchronize")
        return ok


# ------------------------------------------------------------------------------------------ scenes and the oracle

COMB_M = 16


@functools.lru_cache(None)
def scene_arrays(name):
    if name == "comb":
        return LS.comb_scene(COMB_M)[0], LS.COMB_CAM
    return O.Scene.named(name).arrays()


@functools.lru_cache(None)
def oracle_prepared(name, h, w, cam=None):
    s, c = scene_arrays(name)
    return Q.prepare_custom(s, c if cam is None else np.frombuffer(cam, np.float32), h, w)


@functools.lru_cache(None)
def colours(name, h, w, spp, cam=None):
    """float32 [h, w, spp, 3]: the path colour of every sample of every pixel, from the CPU oracle"""
    o = oracle_prepared(name, h, w, cam)
    return o.trace_paths(RB.camera_rays(o.camera(), h, w, spp).reshape(-1, 6))[0].reshape(h, w, spp, 3)


def frame(name, h, w, spp, cam=None):
    """(pixels int32 [h, w], rgb float32 [h, w, 3]) of the frame at spp samples"""
    return frame_of(sequential_sum(colours(name, h, w, spp, cam), 0, spp), spp)


def per_pixel_frame(acc, cnt):
    """frame_of with each pixel's own sample count"""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        rgb = (np.float32(1) / cnt.astype(np.float32))[..., None] * acc
    return quantise(rgb), rgb.astype(np.float32)


def shard_mine(h, w, rank, world):
    tiles_x = (w + 7) // 8
    jj, ii = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return ((jj // 4) * tiles_x + ii // 8) % world == rank


def query_rays(name, n, seed):
    s, _ = scene_arrays(name)
    if name == "comb":
        return LS.comb_query_rays(max(n - 6, 0), seed)[:n]
    return random_rays(s, n, seed)


def ranged_rays(rays6, seed):
    """[n, 8] rays with mixed intervals, one in eleven of them invalid (a NaN t_min or an infinite t_max)"""
    rng = np.random.default_rng(seed)
    n = rays6.shape[0]
    t_min = rng.choice(np.float32([0, 0.1, 1.0, 2.5]), n)
    t_max = rng.choice(np.float32([1e9, 100.0, 7.0, 3.0]), n)
    t_min[::11] = np.nan
    t_max[5::11] = np.inf
    return np.ascontiguousarray(np.concatenate([rays6[:, :3], t_min[:, None], rays6[:, 3:], t_max[:, None]], 1), np.float32)


# ------------------------------------------------------------------------------------------ the GPU side


class Env:
    """A context launching on a torch stream of its own, its prepared scenes, and the hook that runs before every library
    call: nothing, or the poisoning of the pool and of the plain allocator with `pattern`."""

    def __init__(self, **tuning):
        import raytracers_b200 as R
        torch = _torch()
        self.stream = torch.cuda.Stream()
        self.ctx = R.Context(device=0, **tuning)
        self.ctx.set_stream(self.stream.cuda_stream)
        self._prepared = {}
        self.pattern = None
        self.driver = None

    def prepared(self, name, h, w):
        key = (name, h, w)
        if key not in self._prepared:
            self._prepared[key] = self.ctx.prepare_scene(h, w, self.ctx.scene_from_arrays(*scene_arrays(name)))
        return self._prepared[key]

    def before_call(self):
        if self.pattern is None:
            return
        self.ctx.sync()
        assert self.ctx.lib.futhark_context_clear_caches(self.ctx.handle) == 0
        self.driver.poison_plain(self.pattern)
        self.driver.poison_pool(self.stream.cuda_stream, self.pattern)
        assert self.driver.pool_reads_back(self.stream.cuda_stream, self.pattern), \
            f"premise: the pool does not hand out the pattern {self.pattern:#04x} after poisoning"

    def close(self):
        self._prepared.clear()
        self.ctx.close()


# ------------------------------------------------------------------------------------------ the cases
# Each case makes its calls through run_call (guards, inputs), checks what the contract defines against the oracle and
# what it leaves alone against the sentinel, and returns the defined values, which must not depend on the sentinel.


def case_render_into(e, name, h, w, spp, s):
    pr = e.prepared(name, h, w)
    got = run_call(e, lambda p: e.ctx.render_into(p["pix"], h, w, pr, spp, p["rgb"]), {"pix": h * w * 4, "rgb": h * w * 12},
                   sentinel=s, what="render_into")
    pix, rgb = frame(name, h, w, spp)
    assert_equal(as_(got["pix"], np.int32, (h, w)), pix, "render_into pixels")
    assert_bits(as_(got["rgb"], np.float32, (h, w, 3)), rgb, "render_into rgb")
    return got


def case_shards(e, name, h, w, spp, s):
    """render_into and render_shard_into with a shard set, on every rank (a rank may own one tile fewer than the padded
    count, or none), and futhark_entry_render / ray_b200_entry_render_spp's library-owned frames, read back whole."""
    pr = e.prepared(name, h, w)
    want, want_rgb = frame(name, h, w, spp)
    padded = D.tile_layout(h, w, WORLD)[3]
    out = {}
    try:
        for rank in range(WORLD):
            e.ctx.set_shard(rank, WORLD)
            mine = shard_mine(h, w, rank, WORLD)
            got = run_call(e, lambda p: e.ctx.render_into(p["pix"], h, w, pr, spp, p["rgb"]),
                           {"pix": h * w * 4, "rgb": h * w * 12}, sentinel=s, what=f"shard {rank} row-major")
            pix, rgb = as_(got["pix"], np.int32, (h, w)), as_(got["rgb"], np.float32, (h, w, 3))
            assert_equal(pix[mine], want[mine], f"rank {rank} row-major pixels")
            assert_bits(rgb[mine], want_rgb[mine], f"rank {rank} row-major rgb")
            assert_untouched(got["pix"], 4, ~mine, s, f"rank {rank} row-major pixels")
            assert_untouched(got["rgb"], 12, ~mine, s, f"rank {rank} row-major rgb")
            tiles = run_call(e, lambda p: e.ctx.render_shard_into(p["tiles"], h, w, pr, spp), {"tiles": padded * 128},
                             sentinel=s, what=f"shard {rank} tiles")["tiles"]
            assert_equal(as_(tiles, np.int32, (padded, 32)), D.extract_rank_tiles(want, rank, WORLD), f"rank {rank} tiles")
            e.before_call()
            img = e.ctx.render(h, w, pr, spp=None if spp == 1 else spp)
            e.ctx.sync()
            lib = img.values()
            img.free()
            assert_equal(lib, np.where(mine, want, 0), f"rank {rank} library-owned frame")
            out.update({f"{rank} pix": pix[mine], f"{rank} rgb": rgb[mine], f"{rank} tiles": tiles, f"{rank} lib": lib})
    finally:
        e.ctx.set_shard(0, 1)
    e.before_call()
    img = e.ctx.render(h, w, pr, spp=None if spp == 1 else spp)
    e.ctx.sync()
    out["lib"] = img.values()
    img.free()
    assert_equal(out["lib"], want, "library-owned frame")
    return out


def case_batch(e, name, h, w, spp, s):
    pr = e.prepared(name, h, w)
    want, want_rgb = frame(name, h, w, spp)
    padded = D.tile_layout(h, w, WORLD)[3]
    got = run_call(e, lambda p: e.ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=spp, out_dev=p["pix"], out_rgb_dev=p["rgb"]),
                                                    dict(prepared=pr, h=h, w=w, spp=spp, out_dev=p["pix2"])]),
                   {"pix": h * w * 4, "rgb": h * w * 12, "pix2": h * w * 4}, sentinel=s, what="batch")
    assert_equal(as_(got["pix"], np.int32, (h, w)), want, "batch pixels")
    assert_bits(as_(got["rgb"], np.float32, (h, w, 3)), want_rgb, "batch rgb")
    assert_equal(as_(got["pix2"], np.int32, (h, w)), want, "batch second frame")
    try:
        e.ctx.set_shard(WORLD - 1, WORLD)
        tiles = run_call(e, lambda p: e.ctx.render_batch([dict(prepared=pr, h=h, w=w, spp=spp, shard_layout=True, out_dev=p["t"])]),
                         {"t": padded * 128}, sentinel=s, what="batch shard layout")["t"]
    finally:
        e.ctx.set_shard(0, 1)
    assert_equal(as_(tiles, np.int32, (padded, 32)), D.extract_rank_tiles(want, WORLD - 1, WORLD), "batch tiles")
    got["t"] = tiles
    return got


def case_detile(e, name, h, w, spp, s):
    want, _ = frame(name, h, w, spp)
    gathered = np.stack([D.extract_rank_tiles(want, r, WORLD) for r in range(WORLD)])
    got = run_call(e, lambda p: e.ctx.detile(p["g"], p["pix"], h, w, WORLD), {"pix": h * w * 4}, {"g": (gathered, 16)},
                   sentinel=s, what="detile")
    assert_equal(as_(got["pix"], np.int32, (h, w)), want, "detile")
    return got


def case_accumulate(e, name, h, w, spp, s):
    pr = e.prepared(name, h, w)
    col = colours(name, h, w, spp)
    out, acc = {}, h * w * 12
    for a, b in ((0, 1), (1, spp)) if spp > 1 else ((0, 1),):
        got = run_call(e, lambda p: e.ctx.render_accumulate_into(p["acc"], h, w, pr, a, b, p["pix"], p["rgb"]),
                       {"acc": acc, "pix": h * w * 4, "rgb": h * w * 12}, sentinel=s, what=f"accumulate [{a}, {b})")
        want_acc = sequential_sum(col, 0, b)
        want_pix, want_rgb = frame_of(want_acc, b)
        assert_bits(as_(got["acc"], np.float32, (h, w, 3)), want_acc, f"accumulate [{a}, {b}) sums")
        assert_equal(as_(got["pix"], np.int32, (h, w)), want_pix, f"accumulate [{a}, {b}) pixels")
        assert_bits(as_(got["rgb"], np.float32, (h, w, 3)), want_rgb, f"accumulate [{a}, {b}) rgb")
        acc = got["acc"]
        out.update({f"{b} {k}": v for k, v in got.items()})
    return out


def _adaptive(e, name, h, w, spp, s, var):
    """A chain of two calls: every pixel's first sample, then spp more for the pixels of a random mask; with var, the m2
    form and an adaptive_select of the result."""
    pr = e.prepared(name, h, w)
    col = colours(name, h, w, 1 + spp)
    mask = random_masks(h, w, 1, seed=h * 131 + w)[0]
    masks, n_adds = [None, mask], [1, spp]
    out = {}
    bufs = {"acc": h * w * 12, "cnt": np.zeros((h, w), np.int32)}
    if var:
        bufs["m2"] = h * w * 12
    for call, (m, n) in enumerate(zip(masks, n_adds)):
        ins = {} if m is None else {"mask": (m.astype(np.uint8), 16)}

        def go(p):
            if var:
                e.ctx.render_adaptive_var_into(p["acc"], p["m2"], p["cnt"], h, w, pr, n, p.get("mask"), p["pix"], p["rgb"])
            else:
                e.ctx.render_adaptive_into(p["acc"], p["cnt"], h, w, pr, n, p.get("mask"), p["pix"], p["rgb"])
        got = run_call(e, go, {**bufs, "pix": h * w * 4, "rgb": h * w * 12}, ins, sentinel=s, what=f"adaptive call {call}")
        sel = np.ones((h, w), bool) if m is None else m
        if var:
            want_acc, want_m2, want_cnt = m2_model(col, masks[:call + 1], n_adds[:call + 1])
        else:
            want_acc, want_cnt = ragged_model(col, masks[:call + 1], n_adds[:call + 1])
        want_pix, want_rgb = per_pixel_frame(want_acc, want_cnt)
        acc, cnt = as_(got["acc"], np.float32, (h, w, 3)), as_(got["cnt"], np.int32, (h, w))
        pix, rgb = as_(got["pix"], np.int32, (h, w)), as_(got["rgb"], np.float32, (h, w, 3))
        assert_equal(cnt, want_cnt, f"adaptive call {call} counts")
        assert_bits(acc[sel], want_acc[sel], f"adaptive call {call} sums")
        assert_equal(pix[sel], want_pix[sel], f"adaptive call {call} pixels")
        assert_bits(rgb[sel], want_rgb[sel], f"adaptive call {call} rgb")
        assert_untouched(got["pix"], 4, ~sel, s, f"adaptive call {call} unselected pixels")
        assert_untouched(got["rgb"], 12, ~sel, s, f"adaptive call {call} unselected rgb")
        for k, before in bufs.items():    # the sums, M2 and counts of unselected pixels come back as the caller gave them
            if not isinstance(before, int):
                before = np.ascontiguousarray(before).view(np.uint8).reshape(h * w, -1)
                assert np.array_equal(got[k].reshape(h * w, -1)[~sel.reshape(-1)], before[~sel.reshape(-1)]), \
                    f"adaptive call {call}: {k} of an unselected pixel was written"
        if var:
            assert_bits(as_(got["m2"], np.float32, (h, w, 3))[sel], want_m2[sel], f"adaptive call {call} m2")
        out.update({f"{call} acc": acc[sel], f"{call} cnt": cnt, f"{call} pix": pix[sel], f"{call} rgb": rgb[sel]})
        if var:
            out[f"{call} m2"] = as_(got["m2"], np.float32, (h, w, 3))[sel]
        bufs = {k: got[k] for k in bufs}
    if var:
        rule = (0.05, 0.1, 2, 64)
        got = run_call(e, lambda p: e.ctx.adaptive_select_into(p["acc"], p["m2"], p["cnt"], h, w, *rule, p["mask"], p["n"]),
                       {"mask": h * w, "n": 4}, {k: (bufs[k], 16) for k in ("acc", "m2", "cnt")}, sentinel=s, what="adaptive_select")
        want_mask, want_n = select_model(as_(bufs["acc"], np.float32, (h, w, 3)), as_(bufs["m2"], np.float32, (h, w, 3)),
                                         as_(bufs["cnt"], np.int32, (h, w)), *rule)
        assert_equal(got["mask"].reshape(h, w), want_mask.astype(np.uint8), "adaptive_select mask")
        assert int(got["n"].view(np.int32)[0]) == want_n, "adaptive_select n_selected"
        out.update(select_mask=got["mask"], select_n=got["n"])
    return out


def case_adaptive(e, name, h, w, spp, s):
    return _adaptive(e, name, h, w, spp, s, var=False)


def case_adaptive_var(e, name, h, w, spp, s):
    return _adaptive(e, name, h, w, spp, s, var=True)


VIEWS = 7


def case_views(e, name, h, w, spp, s):
    """V views; the host camera table, which the library copies to stream-ordered scratch, comes back unchanged"""
    pr = e.prepared(name, h, w)
    cams = poses(scene_arrays(name)[1], VIEWS, seed=h + 7 * w)
    keep = cams.copy()
    got = run_call(e, lambda p: e.ctx.render_views_into(pr, cams, h, w, spp, p["pix"], p["rgb"]),
                   {"pix": VIEWS * h * w * 4, "rgb": VIEWS * h * w * 12}, sentinel=s, what="views")
    assert np.array_equal(cams.view(np.uint8), keep.view(np.uint8)), "views: the camera table was written"
    for v in range(VIEWS):
        want, want_rgb = frame(name, h, w, spp, cams[v].tobytes())
        assert_equal(as_(got["pix"], np.int32, (VIEWS, h, w))[v], want, f"view {v} pixels")
        assert_bits(as_(got["rgb"], np.float32, (VIEWS, h, w, 3))[v], want_rgb, f"view {v} rgb")
    return got


GB_BYTES = {"id": 4, "depth": 4, "normal": 12, "albedo": 12, "coverage": 4}


@functools.lru_cache(None)
def gbuffer_oracle(name, h, w, spp):
    o = oracle_prepared(name, h, w)
    rays = RB.camera_rays(o.camera(), h, w, spp).reshape(-1, 6)
    g = gbuffer_rule(o.trace_hits(rays), o.trace_paths(rays, max_depth=1)[0], scene_arrays(name)[0][:, 3:6], spp)
    return {k: v.reshape((h, w) + v.shape[1:]) for k, v in g.items()}


def case_gbuffer(e, name, h, w, spp, s, subsets=None):
    pr = e.prepared(name, h, w)
    want = gbuffer_oracle(name, h, w, spp)
    out = {}
    if subsets is None:
        subsets = [c for r in range(1, 6) for c in itertools.combinations(GB_OUTPUTS, r)]
    for names in subsets:
        got = run_call(e, lambda p: e.ctx.render_gbuffer_into(pr, h, w, spp, *(p.get(k, 0) for k in GB_OUTPUTS)),
                       {k: h * w * GB_BYTES[k] for k in names}, sentinel=s, what=f"gbuffer {names}")
        for k in names:
            if k in ("id", "coverage"):
                assert_equal(as_(got[k], np.int32, (h, w)), want[k], f"gbuffer {names}: {k}")
            else:
                assert_bits(got[k].view(np.float32), want[k], f"gbuffer {names}: {k}")
            out[f"{'+'.join(names)} {k}"] = got[k]
    return out


def case_render_host(e, name, h, w, spp, s):
    """render_host: synchronous, through stream-ordered staging frames of the library's own"""
    pr = e.prepared(name, h, w)
    e.before_call()
    pix, rgb = e.ctx.render_host(h, w, pr, spp=spp, want_rgb=True)
    want, want_rgb = frame(name, h, w, spp)
    assert_equal(pix, want, "render_host pixels")
    assert_bits(rgb, want_rgb, "render_host rgb")
    return {"pix": pix, "rgb": rgb}


FRAME_CASES = [case_render_into, case_shards, case_batch, case_detile, case_accumulate, case_adaptive, case_adaptive_var,
               case_views, case_gbuffer, case_render_host]


def case_queries(e, name, n, s, ks=KS, align=16):
    """Every ray query, per-call and ranged, with and without the optional outputs."""
    pr = e.prepared(name, 48, 64)
    o = oracle_prepared(name, 48, 64)
    rays = query_rays(name, n, seed=n)
    r8 = ranged_rays(rays, seed=n + 1)
    ins, ins8 = {"rays": (rays, 16)}, {"rays": (r8, align)}
    c = e.ctx
    out = {}
    got = run_call(e, lambda p: c.trace_hits_into(p["rays"], n, pr, p["hits"], 0.0, 1e9), {"hits": n * 32}, ins, s, "trace_hits")
    assert hits_differ(as_(got["hits"], np.float32, (n, 8)), o.trace_hits(rays)) == 0, "trace_hits"
    out["hits"] = got["hits"]
    want_rgb, want_seg = o.trace_paths(rays)
    got = run_call(e, lambda p: c.trace_paths_into(p["rays"], n, pr, p["rgb"], p["seg"]), {"rgb": n * 12, "seg": n * 4}, ins, s,
                   "trace_paths")
    assert_bits(got["rgb"].view(np.float32), want_rgb, "trace_paths rgb")
    assert_equal(got["seg"].view(np.int32), want_seg, "trace_paths segments")
    got2 = run_call(e, lambda p: c.trace_paths_into(p["rays"], n, pr, p["rgb"], None), {"rgb": n * 12}, ins, s, "trace_paths")
    assert np.array_equal(got2["rgb"], got["rgb"]), "trace_paths without segments"
    out.update(rgb=got["rgb"], seg=got["seg"])
    got = run_call(e, lambda p: c.trace_occluded_into(p["rays"], n, pr, p["occ"], 0.1, 1e9), {"occ": n}, ins, s, "trace_occluded")
    assert_equal(got["occ"], o.trace_occluded(rays, 0.1, 1e9).astype(np.uint8), "trace_occluded")
    out["occ"] = got["occ"]
    got = run_call(e, lambda p: c.trace_hits_ranged_into(p["rays"], n, pr, p["hits"]), {"hits": n * 32}, ins8, s, "hits ranged")
    assert hits_differ(as_(got["hits"], np.float32, (n, 8)), o.trace_hits_ranged(r8)) == 0, "trace_hits_ranged"
    out["hits ranged"] = got["hits"]
    got = run_call(e, lambda p: c.trace_occluded_ranged_into(p["rays"], n, pr, p["occ"]), {"occ": n}, ins8, s, "occluded ranged")
    assert_equal(got["occ"], o.trace_occluded_ranged(r8).astype(np.uint8), "trace_occluded_ranged")
    out["occ ranged"] = got["occ"]
    for k in ks:
        want, want_cnt = o.trace_multi_hits(rays, k)
        got = run_call(e, lambda p: c.trace_multi_hits_into(p["rays"], n, pr, k, p["hits"], p["cnt"]), {"hits": n * k * 32, "cnt": n * 4},
                       ins, s, f"multi k={k}")
        assert hits_differ(as_(got["hits"], np.float32, (n * k, 8)), want.reshape(-1, 8)) == 0, f"trace_multi_hits k={k}"
        assert_equal(got["cnt"].view(np.int32), want_cnt, f"trace_multi_hits k={k} counts")
        got2 = run_call(e, lambda p: c.trace_multi_hits_into(p["rays"], n, pr, k, p["hits"], None), {"hits": n * k * 32}, ins, s,
                        f"multi k={k} no counts")
        assert np.array_equal(got2["hits"], got["hits"]), f"trace_multi_hits k={k} without counts"
        want, want_cnt = o.trace_multi_hits_ranged(r8, k)
        got3 = run_call(e, lambda p: c.trace_multi_hits_ranged_into(p["rays"], n, pr, k, p["hits"], p["cnt"]),
                        {"hits": n * k * 32, "cnt": n * 4}, ins8, s, f"multi ranged k={k}")
        assert hits_differ(as_(got3["hits"], np.float32, (n * k, 8)), want.reshape(-1, 8)) == 0, f"multi ranged k={k}"
        assert_equal(got3["cnt"].view(np.int32), want_cnt, f"multi ranged k={k} counts")
        out.update({f"multi {k}": got["hits"], f"multi {k} cnt": got["cnt"], f"ranged {k}": got3["hits"], f"ranged {k} cnt": got3["cnt"]})
    return out


def case_scene_device(e, name, s, h=33, w=65):
    """prepare_scene_device from 4-byte aligned records, a frame, an update to other records with another n, a frame,
    and prepared_spheres read back: the records are read, never written, and read back as given."""
    sp, cam = scene_arrays(name)
    other = np.ascontiguousarray(sp[::2] if sp.shape[0] >= 4 else np.concatenate([sp, sp + np.float32(3)]), np.float32)
    ctx, out = e.ctx, {}
    holder = {}

    def prep(p):
        holder["pr"] = ctx.prepare_scene_device_from_ptr(h, w, p["s"], sp.shape[0], cam)
    run_call(e, prep, {}, {"s": (sp, 4)}, s, "prepare_scene_device")
    pr = holder["pr"]
    for step, (records, c) in enumerate(((sp, cam), (other, cam))):
        if step:
            run_call(e, lambda p: pr.update_from_ptr(p["s"], records.shape[0]), {}, {"s": (records, 4)}, s, "update")
        want = O.Scene.custom(records, c).prepare(h, w).render(h, w, 3)[0]
        got = run_call(e, lambda p: ctx.render_into(p["pix"], h, w, pr, 3), {"pix": h * w * 4}, sentinel=s, what=f"device scene {step}")
        assert_equal(as_(got["pix"], np.int32, (h, w)), want, f"device-prepared scene, step {step}")
        back = run_call(e, lambda p: ctx._check(ctx.lib.ray_b200_prepared_spheres(ctx.handle, pr.handle, C.c_void_p(p["s"]), None)),
                        {"s": records.nbytes}, sentinel=s, what="prepared_spheres")["s"]
        assert np.array_equal(back, records.view(np.uint8).reshape(-1)), f"prepared_spheres, step {step}"
        out.update({f"{step} pix": got["pix"], f"{step} spheres": back})
    pr.free()
    return out


def assert_same_results(runs, what):
    """The defined values of runs (dicts of arrays) are bit-identical."""
    first = runs[0]
    for r in runs[1:]:
        assert r.keys() == first.keys(), what
        for k in first:
            a, b = np.ascontiguousarray(first[k]), np.ascontiguousarray(r[k])
            assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"{what}: {k} depends on memory contents"


# ------------------------------------------------------------------------------------------ CPU: the helpers


def test_guarded_layout_and_detection():
    torch = _torch()
    for align, nbytes in ((16, 0), (16, 37), (4, 12), (4, 4096)):
        g = Guarded(nbytes, 0xFF, align=align, device="cpu")
        assert g.ptr % 16 == (0 if align == 16 else 4) and g.offset >= GUARD
        assert g.buf.numel() - g.offset - nbytes >= GUARD
        assert (g.buf.numpy() == 0xFF).all()
        assert g.check("fresh").size == nbytes
        if nbytes:
            g.buf[g.offset] = 0
            assert g.check("payload")[0] == 0     # a payload write is not a guard write
        for pos in (g.offset - 1, g.offset + nbytes, 0, g.buf.numel() - 1):
            h = Guarded(nbytes, 0x00, align=align, device="cpu")
            h.buf[pos] = 1
            with pytest.raises(AssertionError, match="written (before|past)"):
                h.check("guard")
    data = np.arange(10, dtype=np.float32)
    g = Guarded(0, 0x7F, align=4, device="cpu", data=data)
    assert g.nbytes == 40 and np.array_equal(g.check("data").view(np.float32), data)
    assert (g.buf[:g.offset].numpy() == 0x7F).all()
    for bad in (dict(sentinel=256), dict(sentinel=-1), dict(sentinel=1.0), dict(align=8), dict(guard=1024), dict(guard=4100),
                dict(nbytes=-1)):
        with pytest.raises(ValueError):
            Guarded(**{"nbytes": 8, "sentinel": 0, "device": "cpu", **bad})
    assert g.buf.dtype == torch.uint8


def test_untouched_and_sameness_helpers():
    p = np.full(24, 0xFF, np.uint8)
    p[4:8] = 0
    assert_untouched(p, 4, np.array([True, False, True, True, True, True]), 0xFF, "ok")
    with pytest.raises(AssertionError, match="1 elements"):
        assert_untouched(p, 4, np.ones(6, bool), 0xFF, "bad")
    a = {"x": np.float32([1, np.nan]), "y": np.int32([3])}
    assert_same_results([a, {k: v.copy() for k, v in a.items()}], "same")
    other_nan = a["x"].copy()
    other_nan.view(np.uint32)[1] ^= 1
    with pytest.raises(AssertionError, match="x depends"):
        assert_same_results([a, {"x": other_nan, "y": a["y"]}], "another NaN payload")


def test_poison_arguments():
    assert poison_args(0, [1]) == (0, [1])
    assert poison_args(np.uint8(255), (4096, 512)) == (255, [4096, 512])
    for bad in (-1, 256, 1.5, True, "0x7f", None):
        with pytest.raises(ValueError, match="pattern"):
            poison_args(bad, [16])
    for bad in ([], [0], [16, -4]):
        with pytest.raises(ValueError, match="sizes"):
            poison_args(0x7F, bad)
    assert all(s > 0 for s in _POOL_FILL + _PLAIN_FILL + _PREMISE)
    assert _POOL_FILL[0] >= 256 << 20, "one large block, for the frames and tables of the sweep"


def test_shard_and_ranged_premises():
    # the shapes cover ranks that own one tile fewer than the padded count, and ranks that own none
    short = [(h, w) for h, w in SHAPES if any(D.rank_tile_count(h, w, r, WORLD) < D.tile_layout(h, w, WORLD)[3] for r in range(WORLD))]
    assert len(short) >= 3
    assert any(D.rank_tile_count(h, w, r, WORLD) == 0 for h, w in SHAPES for r in range(WORLD))
    m = shard_mine(9, 17, 1, 3)
    assert m.sum() == sum(D.extract_rank_tiles(np.ones((9, 17), np.int32), 1, 3).ravel())
    r8 = ranged_rays(np.zeros((33, 6), np.float32), 1)
    assert np.isnan(r8[::11, 3]).all() and np.isinf(r8[5::11, 7]).all()


# ------------------------------------------------------------------------------------------ GPU (a): guarded outputs


@pytest.fixture(scope="module")
def env():
    e = Env()
    yield e
    e.close()


FRAME_PARAMS = [(n, h, w, spp) for n in SCENE_NAMES for (h, w) in SHAPES for spp in (1, 3)] + [("irreg", 9, 5, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,h,w,spp", FRAME_PARAMS, ids=[f"{n}-{h}x{w}-spp{s}" for n, h, w, s in FRAME_PARAMS])
def test_frames_write_only_their_outputs(env, name, h, w, spp):
    for case in FRAME_CASES:
        runs = [case(env, name, h, w, spp, s) for s in SENTINELS]
        assert_same_results(runs, f"{case.__name__} {name} {h}x{w} spp {spp}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", RAY_COUNTS)
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_queries_write_only_their_outputs(env, name, n):
    runs = [case_queries(env, name, n, s, align=a) for s in SENTINELS for a in (16, 4)]
    assert_same_results(runs, f"queries {name} n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_device_scenes_read_their_records_only(env, name):
    assert_same_results([case_scene_device(env, name, s) for s in SENTINELS], f"device scene {name}")


# ------------------------------------------------------------------------------------------ GPU (b): poisoned scratch

LEARN_H, LEARN_W = 64, 96          # 192 tiles: the learned claim order is recorded (more than 64 tiles)


def _learned_order_frames(e, s, heavy=True):
    """A fresh prepared scene (its build scratch from the poisoned pool), its first frame (records the learned order),
    a frame that replays it, and two frames at spp 4: the first records an order for spp 4 or, where the context
    probes at spp > 1 (heavy), runs the heavy-first probe, which the second then runs again instead of replaying."""
    h, w = LEARN_H, LEARN_W
    sp, cam = scene_arrays("irreg")
    ctx = e.ctx
    e.before_call()
    pr = ctx.prepare_scene(h, w, ctx.scene_from_arrays(sp, cam))
    dump, want_dump = pr.dump(), O.Scene.custom(sp, cam).prepare(h, w).dump()
    for k in ("morton", "perm", "left", "right", "parent", "boxes"):
        assert np.array_equal(np.asarray(dump[k]).view(np.uint8), np.asarray(want_dump[k]).view(np.uint8)), f"prepared {k}"
    out, launches = {}, []
    for label, spp in (("record", 1), ("replay", 1), ("spp 4", 4), ("spp 4 again", 4)):
        before = ctx.launch_count()
        got = run_call(e, lambda p: ctx.render_into(p["pix"], h, w, pr, spp, p["rgb"]), {"pix": h * w * 4, "rgb": h * w * 12},
                       sentinel=s, what=label)
        launches.append(ctx.launch_count() - before)
        assert ctx.last_plan()["kernel"] == RB.KERNELS["warpqueue"] and ctx.last_plan()["query"] == "pixels"
        want, want_rgb = frame("irreg", h, w, spp)
        assert_equal(as_(got["pix"], np.int32, (h, w)), want, f"{label} frame")
        assert_bits(as_(got["rgb"], np.float32, (h, w, 3)), want_rgb, f"{label} rgb")
        out.update({f"{label} {k}": v for k, v in got.items()})
    # premises: a recording frame sorts its costs after the kernel, a replay is the kernel alone, and a heavy-first
    # frame runs its probe and sort before the kernel every time
    assert launches[:3] == [launches[0], 1, launches[2]] and launches[0] > 1 and launches[2] > 1, launches
    assert (launches[3] > 1) == heavy, launches
    pr.free()
    return out


@pytest.fixture(scope="module")
def poison_env():
    e = Env(heavy_first=-1)
    e.driver = Driver(0)
    yield e
    e.pattern = None
    e.close()


SWEEP = [(case_render_into, "irreg", 33, 65, 3), (case_render_into, "comb", 9, 5, 16), (case_shards, "rgbbox", 37, 1, 3),
         (case_shards, "irreg", 33, 65, 1), (case_batch, "irreg", 33, 65, 3), (case_detile, "irreg", 9, 5, 1),
         (case_accumulate, "irreg", 33, 65, 3), (case_adaptive, "irreg", 33, 65, 3), (case_adaptive_var, "rgbbox", 33, 65, 3),
         (case_views, "irreg", 33, 65, 3), (case_views, "comb", 9, 5, 1), (case_render_host, "irreg", 33, 65, 3),
         (case_render_host, "rgbbox", LEARN_H, LEARN_W, 4)]


@pytest.mark.gpu
def test_poisoned_scratch_changes_no_output(poison_env):
    e = poison_env
    runs = {}
    for pattern in PATTERNS:
        e.pattern = pattern
        for case, name, h, w, spp in SWEEP:
            runs.setdefault((case.__name__, name, h, w, spp), []).append(case(e, name, h, w, spp, 0x00))
        runs.setdefault("gbuffer", []).append(case_gbuffer(e, "irreg", 33, 65, 3, 0x00, subsets=[GB_OUTPUTS, ("depth", "coverage")]))
        runs.setdefault("learned order", []).append(_learned_order_frames(e, 0x00))
        runs.setdefault("queries", []).append(case_queries(e, "irreg", 1000, 0x00, ks=(7,), align=4))
        runs.setdefault("device scene", []).append(case_scene_device(e, "rgbbox", 0x00))
    e.pattern = None
    for key, r in runs.items():
        assert len(r) == len(PATTERNS)
        assert_same_results(r, f"poisoned {key}")


# ------------------------------------------------------------------------------------------ GPU (c): schedules


def mixed_sequence(e):
    """Frames at spp 1 and 16, every ray query, a G-buffer, views and an adaptive chain, on one context"""
    out = {}
    for label, (case, name, h, w, spp) in enumerate([(case_render_into, "irreg", 33, 65, 1), (case_render_into, "rgbbox", 33, 65, 16),
                                                      (case_views, "irreg", 9, 5, 3), (case_adaptive_var, "irreg", 33, 65, 3)]):
        out.update({f"{label} {k}": v for k, v in case(e, name, h, w, spp, 0x00).items()})
    out.update({f"g {k}": v for k, v in case_gbuffer(e, "irreg", 33, 65, 3, 0x00, subsets=[GB_OUTPUTS]).items()})
    out.update({f"q {k}": v for k, v in case_queries(e, "irreg", 1000, 0x00, ks=(1, 7)).items()})
    return out


@pytest.mark.gpu
def test_two_contexts_on_two_threads():
    envs = [Env(), Env(heavy_first=-1)]
    try:
        serial = [mixed_sequence(e) for e in envs]
        results, errors = [[], []], []

        def work(i):
            try:
                _torch().cuda.set_device(0)
                for _ in range(3):
                    results[i].append(mixed_sequence(envs[i]))
            except BaseException as ex:   # reported by the main thread
                errors.append(ex)
        threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        for i in range(2):
            assert_same_results([serial[i]] + results[i], f"context {i} on its own thread")
    finally:
        for e in envs:
            e.close()


@pytest.mark.gpu
def test_results_next_to_a_busy_gpu():
    """Every frame and query while chained 8192^2 matmuls on another stream hold SMs: the persistent kernel's CTAs
    start as SMs free up.  Pixel frames are the learned-order and heavy-first frames of a 192-tile frame."""
    torch = _torch()
    e = Env(heavy_first=-1)
    side = torch.cuda.Stream()
    try:
        quiet = [_learned_order_frames(e, 0x00), mixed_sequence(e)]
        a = torch.randn(8192, 8192, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            for _ in range(300):
                a = torch.mm(a, a).clamp_(-1, 1)
        busy = [_learned_order_frames(e, 0x00)]
        assert not side.query(), "premise: the matmuls still run when the pixel frames have been rendered"
        busy.append(mixed_sequence(e))
        assert_same_results([quiet[0], busy[0]], "learned order next to matmuls")
        assert_same_results([quiet[1], busy[1]], "mixed sequence next to matmuls")
    finally:
        side.synchronize()
        e.close()


def _tuned_results(tuning):
    e = Env(**tuning)
    try:
        out, plan = {}, None
        for case, name, h, w, spp in [(case_render_into, "irreg", 33, 65, 1), (case_render_into, "irreg", 33, 65, 16),
                                      (case_render_into, "comb", 37, 1, 3), (case_accumulate, "rgbbox", 33, 65, 3)]:
            out.update({f"{case.__name__} {name} {spp} {k}": v for k, v in case(e, name, h, w, spp, 0xFF).items()})
            plan = plan or e.ctx.last_plan()
        if "heavy_first" not in tuning:
            out.update(_learned_order_frames(e, 0xFF, heavy=False))
        for spp in (1, 4):
            got = run_call(e, lambda p: e.ctx.render_into(p["pix"], LEARN_H, LEARN_W, e.prepared("irreg", LEARN_H, LEARN_W), spp),
                           {"pix": LEARN_H * LEARN_W * 4}, sentinel=0xFF, what=f"{tuning}")
            assert_equal(as_(got["pix"], np.int32, (LEARN_H, LEARN_W)), frame("irreg", LEARN_H, LEARN_W, spp)[0], f"{tuning} spp {spp}")
            out[f"192 tiles {spp}"] = got["pix"]
        out.update({f"q {k}": v for k, v in case_queries(e, "irreg", 1000, 0xFF, ks=(7,)).items()})
        out.update(case_gbuffer(e, "irreg", 33, 65, 3, 0xFF, subsets=[GB_OUTPUTS]))
        return out, plan
    finally:
        e.close()


@pytest.mark.gpu
def test_grids_and_claim_orders():
    base, plan = _tuned_results({})
    planned = plan["warps"]
    assert planned >= 8, plan
    tunings = [dict(wq_warps=n) for n in range(1, planned + 1)] + [dict(permute=0), dict(permute=0, heavy_first=1)]
    tunings += [dict(heavy_first=p, probe_segments=g) for p in (1, 2, 4) for g in (1, K_MAX_DEPTH)]
    for t in tunings:
        got, p = _tuned_results(t)
        if "wq_warps" in t:
            assert p["warps"] == t["wq_warps"], (t, p)
        base_keys = {k: base[k] for k in got}
        assert_same_results([base_keys, got], f"tuning {t}")
