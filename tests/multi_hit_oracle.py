"""ctypes binding of the multi-hit oracle (tests/multi_hit_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a fresh temporary directory with the same compiler and flags as the
ray-query oracle (tests/ray_query_oracle.py), so a read-only checkout works.  It contains that whole oracle plus the
multi-hit query; its handles are its own.  Used by tests/test_multi_hits.py, __graft_entry__.smoke() and
tools/bench_rays.py.
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import ray_query_oracle as Q

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "multi_hit_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="multi_hit_oracle_")
        try:
            out = os.path.join(tmp, "libmulti_hit_oracle.so")
            subprocess.check_call([Q._CXX, *Q._FLAGS, "-I", _HERE, "-o", out, _SRC])
            L = C.CDLL(out)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)   # the loaded library stays mapped
        vp, i64, i32, u64, f32 = C.c_void_p, C.c_int64, C.c_int32, C.c_uint64, C.c_float
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
        L.oracle_prepared_dump.argtypes = [vp] * 8
        L.oracle_trace_hits.restype = C.c_int
        L.oracle_trace_hits.argtypes = [vp, vp, i64, f32, f32, vp, i32]
        L.oracle_trace_multi_hits.restype = C.c_int
        L.oracle_trace_multi_hits.argtypes = [vp, vp, i64, f32, f32, i32, vp, vp, i32]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Prepared:
    """`prepared_scene` (ray.fut:239) of the oracle, with the multi-hit query and, to relate the two, objs_hit."""

    def __init__(self, scene_handle, h, w):
        L = lib()
        self._h = L.oracle_prepare_scene(int(h), int(w), scene_handle)
        L.oracle_scene_free(scene_handle)
        if not self._h:
            raise RuntimeError("oracle: prepare_scene failed (needs >= 2 spheres)")

    def trace_multi_hits(self, rays, k, t_min=0.0, t_max=1e9, threads=0):
        """The multi-hit query of every ray of float32[n][6]: (float32[n][k][8] records as struct ray_b200_hit, int32[n]
        counts).  The records are the leaves the bvh_fold walk (bvh.fut:61-84, boxes against (t_min, t_max)) reaches
        whose sphere_hit L[i] r t_min t_max (ray.fut:32-51) is a hit, stable-sorted by (t, leaf), the first k of them;
        empty records (t = -1, sphere = -1, p = normal = 0) after the last.  counts = all accepted leaves."""
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        out = np.empty((r.shape[0], int(k), 8), np.float32)
        counts = np.empty(r.shape[0], np.int32)
        if lib().oracle_trace_multi_hits(self._h, _p(r), r.shape[0], float(t_min), float(t_max), int(k), _p(out), _p(counts),
                                         int(threads)) != 0:
            raise RuntimeError("oracle_trace_multi_hits failed")
        return out, counts

    def trace_hits(self, rays, t_min=0.0, t_max=1e9, threads=0):
        """objs_hit (ray.fut:76-86) of every ray: float32[n][8] records as ray_query_oracle.Prepared.trace_hits."""
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        out = np.empty((r.shape[0], 8), np.float32)
        if lib().oracle_trace_hits(self._h, _p(r), r.shape[0], float(t_min), float(t_max), _p(out), int(threads)) != 0:
            raise RuntimeError("oracle_trace_hits failed")
        return out

    def perm(self, n_spheres):
        """Morton-sorted leaf -> index into the scene's sphere array (the scene has n_spheres spheres)."""
        perm = np.empty(int(n_spheres), np.int32)
        lib().oracle_prepared_dump(self._h, None, _p(perm), None, None, None, None, None)
        return perm

    def camera(self):
        """The 12 camera floats (origin, llc, horizontal, vertical, ray.fut:88-91)."""
        cam = np.empty(12, np.float32)
        lib().oracle_prepared_dump(self._h, None, None, None, None, None, None, _p(cam))
        return cam

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
