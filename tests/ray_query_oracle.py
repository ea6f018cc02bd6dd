"""ctypes binding of the ray-query oracle (tests/ray_query_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a fresh temporary directory with oracle/Makefile's flags, so a read-only
checkout works.  It contains the whole CPU oracle (oracle/oracle.cpp, included unchanged) plus objs_hit / ray_colour for
caller-supplied rays; its handles are its own, not liboracle.so's.  Used by tests/test_ray_queries.py,
__graft_entry__.smoke() and tools/bench_rays.py.
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ray_query_oracle.cpp")
_CXX = "/usr/bin/g++"
_FLAGS = ["-O2", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-shared"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="ray_query_oracle_")
        try:
            out = os.path.join(tmp, "libray_query_oracle.so")
            subprocess.check_call([_CXX, *_FLAGS, "-o", out, _SRC])
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
        L.oracle_render.restype = C.c_int
        L.oracle_render.argtypes = [vp, i64, i64, i32, vp, vp, i32, i32, i32, vp]
        L.oracle_trace_hits.restype = C.c_int
        L.oracle_trace_hits.argtypes = [vp, vp, i64, f32, f32, vp, i32]
        L.oracle_trace_paths.restype = C.c_int
        L.oracle_trace_paths.argtypes = [vp, vp, i64, i32, vp, vp, i32]
        L.oracle_camera_ray.argtypes = [vp, i64, i64, i32, i64, i64, i32, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Prepared:
    """`prepared_scene` (ray.fut:239) of the oracle, with the ray queries."""

    def __init__(self, scene_handle, h, w):
        L = lib()
        self._h = L.oracle_prepare_scene(int(h), int(w), scene_handle)
        L.oracle_scene_free(scene_handle)
        if not self._h:
            raise RuntimeError("oracle: prepare_scene failed (needs >= 2 spheres)")

    def trace_hits(self, rays, t_min=0.0, t_max=1e9, threads=0):
        """objs_hit (ray.fut:76-86) of every ray of float32[n][6]: float32[n][8] records t, bits(sphere), p, normal
        (struct ray_b200_hit; sphere = index into the scene's sphere array, t = sphere = -1 for no hit)."""
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        out = np.empty((r.shape[0], 8), np.float32)
        if lib().oracle_trace_hits(self._h, _p(r), r.shape[0], float(t_min), float(t_max), _p(out), int(threads)) != 0:
            raise RuntimeError("oracle_trace_hits failed")
        return out

    def trace_paths(self, rays, max_depth=50, threads=0):
        """ray_colour (ray.fut:126-148) of every ray of float32[n][6]: (rgb float32[n][3], objs_hit calls int32[n])."""
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        rgb = np.empty((r.shape[0], 3), np.float32)
        seg = np.empty(r.shape[0], np.int32)
        if lib().oracle_trace_paths(self._h, _p(r), r.shape[0], int(max_depth), _p(rgb), _p(seg), int(threads)) != 0:
            raise RuntimeError("oracle_trace_paths failed")
        return rgb, seg

    def camera_ray(self, h, w, j, i, s=0, spp=1):
        """get_ray (ray.fut:109-114) for sample s of pixel (row j, column i) of an h x w frame, as render makes it."""
        out = np.empty(6, np.float32)
        lib().oracle_camera_ray(self._h, int(h), int(w), int(spp), int(j), int(i), int(s), _p(out))
        return out

    def camera(self):
        """The 12 camera floats (origin, llc, horizontal, vertical, ray.fut:88-91)."""
        cam = np.empty(12, np.float32)
        lib().oracle_prepared_dump(self._h, None, None, None, None, None, None, _p(cam))
        return cam

    def perm(self, n):
        out = np.empty(n, np.int32)
        lib().oracle_prepared_dump(self._h, None, _p(out), None, None, None, None, None)
        return out

    def render(self, h, w):
        """oracle_render at 1 spp: (pixels int32[h][w], segments = objs_hit calls of the frame)."""
        pix = np.zeros((h, w), np.int32)
        cnt = (C.c_uint64 * 4)()
        if lib().oracle_render(self._h, int(h), int(w), 1, _p(pix), None, 0, 1, 0, C.byref(cnt)) != 0:
            raise RuntimeError("oracle_render failed")
        return pix, int(cnt[0])

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
