"""ctypes binding of the oracle of the ray queries whose rays carry their own interval (tests/ray_interval_oracle.cpp).
TEST INFRASTRUCTURE ONLY.

Rays are float32[n][8] = struct ray_b200_ray (origin, t_min, direction, t_max).  Each answer is that of the per-call
query of tests/ray_query_oracle.py for the ray alone with its (t_min, t_max); a ray whose interval the per-call entry
points reject (t_min not finite and >= 0, t_max not finite) gets the empty answer, as the library defines it.  The
library is compiled on first use into a fresh temporary directory with the ray-query oracle's flags, so a read-only
checkout works; its handles are its own.  Used by tests/test_ray_intervals.py, __graft_entry__.smoke() and
tools/bench_rays.py.
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import ray_query_oracle as _Q

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ray_interval_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="ray_interval_oracle_")
        try:
            out = os.path.join(tmp, "libray_interval_oracle.so")
            subprocess.check_call([_Q._CXX, *_Q._FLAGS, "-o", out, _SRC])
            L = C.CDLL(out)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)   # the loaded library stays mapped
        vp, i64, i32, u64 = C.c_void_p, C.c_int64, C.c_int32, C.c_uint64
        L.oracle_scene_rgbbox.restype = vp
        L.oracle_scene_irreg.restype = vp
        L.oracle_scene_random.restype = vp
        L.oracle_scene_random.argtypes = [i64, u64]
        L.oracle_scene_custom.restype = vp
        L.oracle_scene_custom.argtypes = [vp, i64, vp]
        L.oracle_scene_free.argtypes = [vp]
        L.oracle_prepare_scene.restype = vp
        L.oracle_prepare_scene.argtypes = [i64, i64, vp]
        L.oracle_prepared_free.argtypes = [vp]
        L.oracle_trace_hits_ranged.restype = C.c_int
        L.oracle_trace_hits_ranged.argtypes = [vp, vp, i64, vp, i32]
        L.oracle_trace_occluded_ranged.restype = C.c_int
        L.oracle_trace_occluded_ranged.argtypes = [vp, vp, i64, vp, i32]
        L.oracle_trace_multi_hits_ranged.restype = C.c_int
        L.oracle_trace_multi_hits_ranged.argtypes = [vp, vp, i64, i32, vp, vp, i32]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rays8(rays8):
    return np.ascontiguousarray(rays8, np.float32).reshape(-1, 8)


class Prepared:
    """`prepared_scene` (ray.fut:239) of the oracle, with the ranged ray queries."""

    def __init__(self, scene_handle, h, w):
        L = lib()
        self._h = L.oracle_prepare_scene(int(h), int(w), scene_handle)
        L.oracle_scene_free(scene_handle)
        if not self._h:
            raise RuntimeError("oracle: prepare_scene failed (needs >= 2 spheres)")

    def trace_hits_ranged(self, rays8, threads=0):
        """objs_hit of every ray with its own interval: float32[n][8] records as struct ray_b200_hit."""
        r = _rays8(rays8)
        out = np.empty((r.shape[0], 8), np.float32)
        if lib().oracle_trace_hits_ranged(self._h, _p(r), r.shape[0], _p(out), int(threads)) != 0:
            raise RuntimeError("oracle_trace_hits_ranged failed")
        return out

    def trace_occluded_ranged(self, rays8, threads=0):
        """Occlusion of every ray with its own interval: bool[n]."""
        r = _rays8(rays8)
        out = np.empty(r.shape[0], np.uint8)
        if lib().oracle_trace_occluded_ranged(self._h, _p(r), r.shape[0], _p(out), int(threads)) != 0:
            raise RuntimeError("oracle_trace_occluded_ranged failed")
        return out.view(np.bool_)

    def trace_multi_hits_ranged(self, rays8, k, threads=0):
        """The multi-hit query of every ray with its own interval: (float32[n][k][8] records, int32[n] counts)."""
        r = _rays8(rays8)
        out = np.empty((r.shape[0], int(k), 8), np.float32)
        counts = np.empty(r.shape[0], np.int32)
        if lib().oracle_trace_multi_hits_ranged(self._h, _p(r), r.shape[0], int(k), _p(out), _p(counts), int(threads)) != 0:
            raise RuntimeError("oracle_trace_multi_hits_ranged failed")
        return out, counts

    def __del__(self):
        if getattr(self, "_h", None):
            lib().oracle_prepared_free(self._h)
            self._h = None


def prepare(name, h, w, n=None, seed=1):
    """A built-in scene ("rgbbox", "irreg", "random" with n spheres) prepared for an h x w frame."""
    L = lib()
    s = {"rgbbox": L.oracle_scene_rgbbox, "irreg": L.oracle_scene_irreg}.get(name)
    handle = s() if s else L.oracle_scene_random(int(n), int(seed))
    return Prepared(handle, h, w)


def prepare_custom(spheres, cam7, h, w):
    s = np.ascontiguousarray(spheres, np.float32).reshape(-1, 7)
    c = np.ascontiguousarray(cam7, np.float32).reshape(7)
    return Prepared(lib().oracle_scene_custom(_p(s), s.shape[0], _p(c)), h, w)
