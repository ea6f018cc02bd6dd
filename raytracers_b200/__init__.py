"""raytracers_b200 — host-side mirror of the reference's Futhark entry points over libray_b200.so.

The reference's public surface for the render path is four Futhark entries (futhark/ray.fut:176,
223, 241, 246) reached through the generated C API that futhark/main.c calls (main.c:59-141).  This
module binds the same C ABI (include/ray.h, include/ray_b200.h) with ctypes and exposes the same
names with the same argument order and error behaviour:

    ctx = Context()
    scene = ctx.rgbbox()                      # entry rgbbox        (ray.fut:176)
    prepared = ctx.prepare_scene(h, w, scene) # entry prepare_scene (ray.fut:241)  note (h, w)
    img = ctx.render(h, w, prepared)          # entry render        (ray.fut:246)  -> Image [h][w] i32
    ctx.sync(); pixels = img.values()         # futhark_context_sync / futhark_values_i32_2d

All compute happens in hand-written sm_90a CUDA kernels inside the shared library.  There is no
Python or CPU fallback: if the library is missing or no H100 is visible, Context() raises.
This package never imports anything from oracle/.
"""
import ctypes as C
import os

import numpy as np

__all__ = ["Context", "RayError", "Hit", "Ray", "Ball", "Near", "proximity_k", "proximity_balls", "nearest_k", "nearest_points", "Plan", "QUERIES", "lib_path", "load_library", "KERNELS", "declared_symbols", "host_scene",
           "host_camera", "host_lbvh", "host_sample_offsets", "camera_table", "camera_rays", "SceneBatch", "scene_batch_rows",
           "scene_batch_counts", "scene_batch_cameras", "scene_batch_frames_ok"]

_HERE = os.path.dirname(os.path.abspath(__file__))
KERNELS = {"auto": 0, "mega": 1, "persistent": 2, "wavefront": 3, "warpqueue": 4, "streamqueue": 5, "lanewalk": 6}
# The measured-slower alternative kernels are not part of the product library: they live in libray_b200_all.so (the
# same objects + render_alt_kernels.cu built with RAYB200_ALL_KERNELS), which Context() loads when one of them is named.
ALT_KERNELS = {2, 3, 5, 6}


class RayError(RuntimeError):
    pass


def lib_path(variant=""):
    # RAY_B200_LIB: load another build of the same library (development A/B runs only)
    if variant == "all":
        return os.path.join(_HERE, "libray_b200_all.so")
    return os.environ.get("RAY_B200_LIB") or os.path.join(_HERE, "libray_b200.so")


class BvhInfo(C.Structure):
    _fields_ = [("n_leaves", C.c_int64), ("n_inner", C.c_int64), ("max_depth", C.c_int32), ("refit_sweeps", C.c_int32),
                ("stale_nodes", C.c_int32), ("smem_nodes", C.c_int32), ("root_box", C.c_float * 6),
                ("camera", C.c_float * 12)]


class WorkCounters(C.Structure):
    _fields_ = [("segments", C.c_uint64), ("node_steps", C.c_uint64), ("box_tests", C.c_uint64),
                ("leaf_tests", C.c_uint64)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class Plan(C.Structure):
    """struct ray_b200_plan (include/ray_b200.h): the plan of the last render kernel launch on a context, 80 bytes."""
    _fields_ = [("kernel", C.c_int32), ("query", C.c_int32), ("ranged", C.c_int32), ("k", C.c_int32), ("warps", C.c_int32),
                ("ctas", C.c_int32), ("spread", C.c_int32), ("packet", C.c_int32), ("all_nodes", C.c_int32),
                ("spheres", C.c_int32), ("ncap", C.c_int32), ("nlow", C.c_int32), ("smem_nodes", C.c_int32),
                ("smem_spheres", C.c_int32), ("n_inner", C.c_int32), ("n_leaves", C.c_int32), ("stage_budget", C.c_int64),
                ("dynamic_smem", C.c_int64)]


# enum ray_b200_query: what a launch traces (Plan.query)
QUERIES = ("pixels", "closest", "anyhit", "multihit", "accumulate", "views", "adaptive", "adaptive_var", "gbuffer", "scene_batch",
           "scene_batch_closest", "scene_batch_anyhit", "scene_batch_multihit")


class RenderJob(C.Structure):
    """struct ray_b200_render_job (include/ray_b200.h)."""
    _fields_ = [("prepared", C.c_void_p), ("h", C.c_int64), ("w", C.c_int64), ("spp", C.c_int32), ("shard_layout", C.c_int32),
                ("out_dev", C.c_void_p), ("out_rgb_dev", C.c_void_p), ("wait_flag", C.c_void_p), ("wait_value", C.c_uint32),
                ("reserved0", C.c_uint32), ("done_flag", C.c_void_p)]


class Hit(C.Structure):
    """struct ray_b200_hit (include/ray_b200.h): the closest hit of one ray, 32 bytes."""
    _fields_ = [("t", C.c_float), ("sphere", C.c_int32), ("p", C.c_float * 3), ("normal", C.c_float * 3)]


class Ray(C.Structure):
    """struct ray_b200_ray (include/ray_b200.h): a ray with its own interval, 32 bytes; the rows of an [n, 8] float32
    tensor of rays (origin, t_min, direction, t_max)."""
    _fields_ = [("o", C.c_float * 3), ("t_min", C.c_float), ("d", C.c_float * 3), ("t_max", C.c_float)]


class Ball(C.Structure):
    """struct ray_b200_ball (include/ray_b200.h): a proximity query, centre and radius, 16 bytes; the rows of an [n, 4]
    float32 tensor of balls."""
    _fields_ = [("c", C.c_float * 3), ("r", C.c_float)]


class Near(C.Structure):
    """struct ray_b200_near (include/ray_b200.h): one sphere within a ball, signed distance d and caller index, 8 bytes."""
    _fields_ = [("d", C.c_float), ("sphere", C.c_int32)]


_libs = {}


def _or(value, default):
    return default if value is None else value


def load_library(variant=""):
    """Loads libray_b200.so (built by `make -C raytracers_b200/csrc` / __graft_entry__.build()); variant "all" =
    libray_b200_all.so, the build that also carries the alternative kernels K1 / K2 / K4."""
    if variant in _libs:
        return _libs[variant]
    path = lib_path(variant)
    if not os.path.exists(path):
        raise RayError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no fallback implementation)")
    L = C.CDLL(path)
    vp, i64, i32, u64 = C.c_void_p, C.c_int64, C.c_int32, C.c_uint64
    pp = C.POINTER(vp)
    sig = {
        "futhark_context_config_new": (vp, []),
        "futhark_context_config_free": (None, [vp]),
        "futhark_context_config_set_debugging": (None, [vp, C.c_int]),
        "futhark_context_config_set_profiling": (None, [vp, C.c_int]),
        "futhark_context_config_set_logging": (None, [vp, C.c_int]),
        "futhark_context_config_set_device": (None, [vp, C.c_char_p]),
        "futhark_context_config_set_tuning_param": (C.c_int, [vp, C.c_char_p, C.c_size_t]),
        "futhark_get_tuning_param_count": (C.c_int, []),
        "futhark_get_tuning_param_name": (C.c_char_p, [C.c_int]),
        "futhark_context_new": (vp, [vp]),
        "futhark_context_free": (None, [vp]),
        "futhark_context_sync": (C.c_int, [vp]),
        "futhark_context_get_error": (vp, [vp]),
        "futhark_context_report": (vp, [vp]),
        "futhark_context_clear_caches": (C.c_int, [vp]),
        "futhark_new_i32_2d": (vp, [vp, vp, i64, i64]),
        "futhark_new_raw_i32_2d": (vp, [vp, vp, i64, i64]),
        "futhark_free_i32_2d": (C.c_int, [vp, vp]),
        "futhark_values_i32_2d": (C.c_int, [vp, vp, vp]),
        "futhark_values_raw_i32_2d": (vp, [vp, vp]),
        "futhark_shape_i32_2d": (C.POINTER(i64), [vp, vp]),
        "futhark_free_opaque_scene": (C.c_int, [vp, vp]),
        "futhark_store_opaque_scene": (C.c_int, [vp, vp, pp, C.POINTER(C.c_size_t)]),
        "futhark_restore_opaque_scene": (vp, [vp, vp]),
        "futhark_free_opaque_prepared_scene": (C.c_int, [vp, vp]),
        "futhark_store_opaque_prepared_scene": (C.c_int, [vp, vp, pp, C.POINTER(C.c_size_t)]),
        "futhark_restore_opaque_prepared_scene": (vp, [vp, vp]),
        "futhark_entry_rgbbox": (C.c_int, [vp, pp]),
        "futhark_entry_irreg": (C.c_int, [vp, pp]),
        "futhark_entry_prepare_scene": (C.c_int, [vp, pp, i64, i64, vp]),
        "futhark_entry_render": (C.c_int, [vp, pp, i64, i64, vp]),
        "ray_b200_context_set_stream": (C.c_int, [vp, vp]),
        "ray_b200_context_set_spp": (C.c_int, [vp, i32]),
        "ray_b200_context_set_kernel": (C.c_int, [vp, i32]),
        "ray_b200_context_set_shard": (C.c_int, [vp, i32, i32]),
        "ray_b200_context_device": (C.c_int, [vp]),
        "ray_b200_context_last_render_ms": (C.c_int, [vp, C.POINTER(C.c_float)]),
        "ray_b200_render_batch": (C.c_int, [vp, C.POINTER(RenderJob), C.c_int32]),
        "ray_b200_render_job_size": (C.c_int64, []),
        "ray_b200_context_set_pipeline": (C.c_int, [vp, i32]),
        "ray_b200_pipeline_join": (C.c_int, [vp]),
        "ray_b200_context_trace_warps": (C.c_int, [vp, C.c_int32]),
        "ray_b200_context_warp_trace": (C.c_int, [vp, C.POINTER(C.c_float), C.c_int64, C.POINTER(C.c_int64)]),
        "ray_b200_context_launch_count": (i64, [vp]),
        "ray_b200_context_last_plan": (C.c_int, [vp, C.POINTER(Plan)]),
        "ray_b200_plan_size": (i64, []),
        "ray_b200_scene_from_arrays": (C.c_int, [vp, pp, vp, i64, vp]),
        "ray_b200_scene_random": (C.c_int, [vp, pp, i64, u64]),
        "ray_b200_scene_num_spheres": (i64, [vp, vp]),
        "ray_b200_scene_get_arrays": (C.c_int, [vp, vp, vp, vp]),
        "ray_b200_prepared_info": (C.c_int, [vp, vp, C.POINTER(BvhInfo)]),
        "ray_b200_prepared_dump": (C.c_int, [vp] * 8),
        "ray_b200_prepared_reupload": (C.c_int, [vp, vp]),
        "ray_b200_prepared_packed": (C.c_int, [vp, vp, vp, vp, vp, vp]),
        "ray_b200_prepared_upload_bytes": (i64, [vp, vp]),
        "ray_b200_prepared_device_bytes": (i64, [vp, vp]),
        "ray_b200_prepare_scene_device": (C.c_int, [vp, pp, i64, i64, vp, i64, vp]),
        "ray_b200_prepared_update": (C.c_int, [vp, vp, vp, i64, vp]),
        "ray_b200_prepared_spheres": (C.c_int, [vp, vp, vp, vp]),
        "ray_b200_render_into": (C.c_int, [vp, vp, vp, i64, i64, i32, vp]),
        "ray_b200_render_host": (C.c_int, [vp, vp, vp, i64, i64, i32, vp]),
        "ray_b200_render_accumulate": (C.c_int, [vp, vp, i64, i64, i32, i32, vp, vp, vp]),
        "ray_b200_render_adaptive": (C.c_int, [vp, vp, vp, vp, i64, i64, i32, vp, vp, vp]),
        "ray_b200_render_adaptive_var": (C.c_int, [vp, vp, vp, vp, vp, i64, i64, i32, vp, vp, vp]),
        "ray_b200_adaptive_select": (C.c_int, [vp, vp, vp, vp, i64, i64, C.c_float, C.c_float, i32, i32, vp, vp]),
        "ray_b200_render_views_into": (C.c_int, [vp, vp, vp, i32, i64, i64, i32, vp, vp]),
        "ray_b200_render_gbuffer": (C.c_int, [vp, vp, i64, i64, i32, vp, vp, vp, vp, vp]),
        "ray_b200_entry_render_spp": (C.c_int, [vp, pp, i64, i64, i32, vp]),
        "ray_b200_scene_batch_new_device": (C.c_int, [vp, pp, i64, i64, vp, i32, i64, vp]),
        "ray_b200_scene_batch_new_ragged": (C.c_int, [vp, pp, i64, i64, vp, i32, vp, vp]),
        "ray_b200_scene_batch_update": (C.c_int, [vp, vp, vp, vp]),
        "ray_b200_scene_batch_update_ragged": (C.c_int, [vp, vp, vp, vp, vp]),
        "ray_b200_scene_batch_counts": (C.c_int, [vp, vp, vp]),
        "ray_b200_scene_batch_free": (C.c_int, [vp, vp]),
        "ray_b200_scene_batch_shape": (C.c_int, [vp, vp, C.POINTER(i32), C.POINTER(i64)]),
        "ray_b200_scene_batch_member": (C.c_int, [vp, vp, i32, pp]),
        "ray_b200_render_scene_batch_into": (C.c_int, [vp, vp, i64, i64, i32, vp, vp]),
        "ray_b200_scene_batch_trace_hits": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, vp]),
        "ray_b200_scene_batch_trace_paths": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_scene_batch_trace_occluded": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, vp]),
        "ray_b200_scene_batch_trace_multi_hits": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, i32, vp, vp]),
        "ray_b200_scene_batch_trace_hits_ranged": (C.c_int, [vp, vp, vp, i64, vp]),
        "ray_b200_scene_batch_trace_occluded_ranged": (C.c_int, [vp, vp, vp, i64, vp]),
        "ray_b200_scene_batch_trace_multi_hits_ranged": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_shard_tiles": (i64, [i64, i64, i32, i32]),
        "ray_b200_shard_tiles_padded": (i64, [i64, i64, i32]),
        "ray_b200_render_shard_into": (C.c_int, [vp, vp, i64, i64, i32, vp]),
        "ray_b200_detile": (C.c_int, [vp, vp, vp, i64, i64, i32]),
        "ray_b200_trace_hits": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, vp]),
        "ray_b200_trace_paths": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_trace_occluded": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, vp]),
        "ray_b200_trace_multi_hits": (C.c_int, [vp, vp, vp, i64, C.c_float, C.c_float, i32, vp, vp]),
        "ray_b200_hit_size": (i64, []),
        "ray_b200_trace_hits_ranged": (C.c_int, [vp, vp, vp, i64, vp]),
        "ray_b200_trace_occluded_ranged": (C.c_int, [vp, vp, vp, i64, vp]),
        "ray_b200_trace_multi_hits_ranged": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_ray_size": (i64, []),
        "ray_b200_query_spheres": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_scene_batch_query_spheres": (C.c_int, [vp, vp, vp, i64, i32, vp, vp]),
        "ray_b200_query_nearest": (C.c_int, [vp, vp, vp, i64, i32, vp]),
        "ray_b200_scene_batch_query_nearest": (C.c_int, [vp, vp, vp, i64, i32, vp]),
        "ray_b200_near_size": (i64, []),
        "ray_b200_ball_size": (i64, []),
        "ray_b200_count_work": (C.c_int, [vp, i64, i64, i32, vp, C.POINTER(WorkCounters)]),
        "ray_b200_ipc_alloc": (C.c_int, [vp, i64, pp, vp]),
        "ray_b200_ipc_free": (C.c_int, [vp, vp]),
        "ray_b200_ipc_open": (C.c_int, [vp, vp, pp]),
        "ray_b200_ipc_close": (C.c_int, [vp, vp]),
        "ray_b200_flag_wait": (C.c_int, [vp, vp, vp, C.c_uint32, i32]),
        "ray_b200_flag_set": (C.c_int, [vp, vp, vp, C.c_uint32]),
        "ray_b200_flag_status": (C.c_int, [vp, C.POINTER(i64)]),
        "ray_b200_copy_to_host_async": (C.c_int, [vp, vp, vp, vp, i64]),
        "ray_b200_host_scene": (C.c_int, [C.c_char_p, i64, u64, vp, i64, vp, C.POINTER(i64)]),
        "ray_b200_host_camera": (C.c_int, [vp, i64, i64, vp]),
        "ray_b200_host_lbvh": (C.c_int, [vp, i64, vp, vp, vp, vp, vp, vp, vp]),
        "ray_b200_host_sample_offsets": (None, [i32, vp]),
        "ray_b200_version": (C.c_char_p, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)  # AttributeError here = the library does not export what the headers declare
        fn.restype = res
        fn.argtypes = args
    L._declared = tuple(sig)
    _libs[variant] = L
    return L


def declared_symbols():
    """Names this binding expects the library to export (the test suite checks them against include/*.h)."""
    return load_library()._declared


_libc_free = None


def _free(ptr):
    global _libc_free
    if _libc_free is None:
        _libc_free = C.CDLL(None).free
        _libc_free.argtypes = [C.c_void_p]
    _libc_free(ptr)


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))  # raw device/host address (e.g. torch.Tensor.data_ptr())


# ---- host-only helpers (no GPU needed): the setup path's host logic, used by the CPU test suite -----------
def host_scene(name, n=0, seed=1):
    """(spheres[n][7], cam7) of a built-in scene generator (ray.fut:176-237 / the random extension)."""
    L = load_library()
    cnt = C.c_int64(0)
    if L.ray_b200_host_scene(name.encode(), int(n), int(seed), None, 0, None, C.byref(cnt)) != 0:
        raise RayError(f"unknown scene {name!r}")
    s = np.empty((cnt.value, 7), np.float32)
    c = np.empty(7, np.float32)
    if L.ray_b200_host_scene(name.encode(), int(n), int(seed), _ptr(s), cnt.value, _ptr(c), None) != 0:
        raise RayError("host_scene failed")
    return s, c


def host_camera(cam7, h, w):
    out = np.empty(12, np.float32)
    c = np.ascontiguousarray(cam7, np.float32)
    if load_library().ray_b200_host_camera(_ptr(c), int(h), int(w), _ptr(out)) != 0:
        raise RayError("host_camera failed")
    return out


def host_lbvh(spheres):
    """prepare_scene's LBVH (bvh.fut:30-59) in the reference's node order, built by the product's host code."""
    s = np.ascontiguousarray(spheres, np.float32).reshape(-1, 7)
    n = s.shape[0]
    m = max(n - 1, 0)
    out = dict(morton=np.empty(n, np.uint32), perm=np.empty(n, np.int32), left=np.empty(m, np.int32),
               right=np.empty(m, np.int32), parent=np.empty(m, np.int32), boxes=np.empty((m, 6), np.float32))
    info = np.zeros(4, np.int32)
    rc = load_library().ray_b200_host_lbvh(_ptr(s), n, _ptr(out["morton"]), _ptr(out["perm"]), _ptr(out["left"]),
                                           _ptr(out["right"]), _ptr(out["parent"]), _ptr(out["boxes"]), _ptr(info))
    if rc == 2:
        raise RayError("prepare_scene: a scene needs at least 2 spheres")
    if rc != 0:
        raise RayError("host_lbvh failed")
    out.update(refit_sweeps=int(info[0]), max_depth=int(info[1]), stale_nodes=int(info[2]))
    return out


def host_sample_offsets(spp):
    t = np.empty((spp, 2), np.float32)
    load_library().ray_b200_host_sample_offsets(int(spp), _ptr(t))
    return t


def camera_table(cams):
    """The cameras of Context.render_views as the library reads them: a contiguous float32 [V, 7] array (look_from.xyz,
    look_at.xyz, fov of each view) from any host array-like of shape [V, 7] with a floating-point dtype.  A CUDA tensor
    raises ValueError (reading it would synchronise the device), and so does any other shape or dtype."""
    if type(cams).__module__.startswith("torch"):
        if cams.device.type != "cpu":
            raise ValueError(f"cams must be a host array of shape [V, 7], got a tensor on {cams.device}")
        cams = cams.numpy()
    a = np.asarray(cams)
    if a.ndim != 2 or a.shape[1] != 7:
        raise ValueError(f"cams must have shape [V, 7], got {a.shape}")
    if a.dtype.kind != "f":
        raise ValueError(f"cams must be floating-point, got {a.dtype}")
    return np.ascontiguousarray(a, np.float32)


def _check_tensor(device, name, t, dtypes, shape):
    """ValueError unless t is a contiguous CUDA tensor on cuda:device of one of dtypes and of this shape"""
    import torch
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda" or t.device.index != device:
        raise ValueError(f"{name} must be a CUDA tensor on cuda:{device}")
    if t.dtype not in dtypes or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous {'/'.join(str(d) for d in dtypes)} tensor of shape {list(shape)}, "
                         f"got {t.dtype} {tuple(t.shape)}")


def _sphere_rows(device, spheres):
    """n of spheres, a contiguous float32 CUDA tensor [n, 7] on cuda:device; ValueError for anything else"""
    import torch
    if not isinstance(spheres, torch.Tensor) or spheres.dim() != 2:
        raise ValueError("spheres must be a float32 CUDA tensor of shape [n, 7]")
    _check_tensor(device, "spheres", spheres, (torch.float32,), (spheres.shape[0], 7))
    return int(spheres.shape[0])


def scene_batch_rows(device, spheres):
    """(B, n) of spheres, a contiguous float32 CUDA tensor [B, n, 7] on cuda:device with B >= 1, 2 <= n and B n <= 2^26;
    ValueError for anything else"""
    import torch
    if not isinstance(spheres, torch.Tensor) or spheres.dim() != 3:
        raise ValueError("spheres must be a float32 CUDA tensor of shape [B, n, 7]")
    B, n = int(spheres.shape[0]), int(spheres.shape[1])
    _check_tensor(device, "spheres", spheres, (torch.float32,), (B, n, 7))
    if B < 1 or n < 2:
        raise ValueError(f"a scene batch needs B >= 1 scenes of n >= 2 spheres, got B = {B}, n = {n}")
    if B * n > 1 << 26:
        raise ValueError(f"a scene batch holds at most 2^26 spheres, got {B} x {n}")
    return B, n


def scene_batch_counts(device, spheres, counts, B=None):
    """(B, counts) of a ragged scene batch: counts, B >= 1 host integers (a sequence, array or CPU tensor; B of them when
    B is given, as for an update), each >= 2 and summing to N <= 2^26, as a contiguous int64 array, and spheres, a
    contiguous float32 CUDA tensor [N, 7] on cuda:device (scene b's records from row counts[0] + .. + counts[b - 1]);
    ValueError for anything else.  The counts are checked first, on the host."""
    import torch
    if isinstance(counts, torch.Tensor):
        if counts.device.type != "cpu":
            raise ValueError("counts must be on the host (reading a CUDA tensor would synchronise the device)")
        counts = counts.numpy()
    c = np.asarray(counts) if counts is not None else np.zeros((0,), np.float32)
    if c.ndim != 1 or len(c) < 1 or c.dtype.kind not in "iu":
        raise ValueError(f"counts must be a 1-d sequence of B >= 1 integers, got {c.dtype} {c.shape}")
    if B is not None and len(c) != B:
        raise ValueError(f"counts must hold the batch's {B} counts, got {len(c)}")
    if int(c.min()) < 2:
        raise ValueError(f"every scene of a batch needs at least 2 spheres, got a count of {int(c.min())}")
    if int(c.max()) > 1 << 26 or int(c.astype(np.int64).sum()) > 1 << 26:
        raise ValueError("a scene batch holds at most 2^26 spheres, the counts sum to more")
    c = np.ascontiguousarray(c, np.int64)
    N = int(c.sum())
    if not isinstance(spheres, torch.Tensor) or spheres.dim() != 2 or int(spheres.shape[0]) != N:
        raise ValueError(f"spheres must be a float32 CUDA tensor of shape [N, 7] with N = sum(counts) = {N}, got "
                         f"{tuple(spheres.shape) if isinstance(spheres, torch.Tensor) else type(spheres).__name__}")
    _check_tensor(device, "spheres", spheres, (torch.float32,), (N, 7))
    return len(c), c


def scene_batch_cameras(cams, B):
    """cams as the contiguous float32 host [B, 7] array the batch calls read, from a host array-like or a tensor of shape
    [B, 7] with a floating-point dtype (a CUDA tensor is copied to the host, which synchronises); ValueError otherwise."""
    if type(cams).__module__.startswith("torch"):
        cams = cams.detach().cpu().numpy()
    a = np.asarray(cams)
    if a.shape != (B, 7) or a.dtype.kind != "f":
        raise ValueError(f"cams must have shape [{B}, 7] and a floating-point dtype, got {a.dtype} {a.shape}")
    return np.ascontiguousarray(a, np.float32)


def scene_batch_frames_ok(B, h, w):
    """Whether B frames of h x w fit one launch: h, w in [1, 65536] and B x ceil(h / 4) x ceil(w / 8) <= 2^25 tiles"""
    return 0 < h <= 65536 and 0 < w <= 65536 and B * ((h + 3) // 4) * ((w + 7) // 8) <= 1 << 25


def proximity_k(k):
    """k of a proximity query, an integer in [0, 64] (0: count only); ValueError otherwise"""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= int(k) <= 64:
        raise ValueError(f"k must be an integer in [0, 64], got {k!r}")
    return int(k)


def proximity_balls(device, balls, B=None):
    """The balls of a proximity query: a contiguous float32 CUDA tensor on cuda:device of shape [n, 4] (centre.xyz, r), or
    with B (a scene batch's) [B, m, 4] with B m <= 2^30.  Returns n, or m for a batch; ValueError for anything else,
    including spheres' own [n, 7] rows (make balls of them with torch.cat([s[:, :3], s[:, 6:7]], 1))."""
    import torch
    dims = 2 if B is None else 3
    shape = "[n, 4]" if B is None else "[B, m, 4]"
    if not isinstance(balls, torch.Tensor) or balls.dim() != dims or balls.shape[-1] != 4:
        got = f"{balls.dtype} {tuple(balls.shape)}" if isinstance(balls, torch.Tensor) else type(balls).__name__
        raise ValueError(f"balls must be a float32 CUDA tensor of shape {shape} (centre.xyz, r), got {got}")
    _check_tensor(device, "balls", balls, (torch.float32,), tuple(balls.shape))
    if B is None:
        if balls.shape[0] > 1 << 30:
            raise ValueError(f"a proximity query takes at most 2^30 balls, got {balls.shape[0]}")
        return int(balls.shape[0])
    if int(balls.shape[0]) != B:
        raise ValueError(f"balls must have one row per scene of the batch ({B}), got {int(balls.shape[0])}")
    if B * int(balls.shape[1]) > 1 << 30:
        raise ValueError(f"a batch proximity query takes at most 2^30 balls, got {B} x {int(balls.shape[1])}")
    return int(balls.shape[1])


def nearest_k(k):
    """k of a nearest-sphere query, an integer in [1, 64]; ValueError otherwise"""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= 64:
        raise ValueError(f"k must be an integer in [1, 64], got {k!r}")
    return int(k)


def nearest_points(device, points, B=None):
    """The balls of a nearest-sphere query from points, a contiguous float32 CUDA tensor on cuda:device of shape [n, 3]
    (centres, no limit on the distance) or [n, 4] (centre.xyz, r), or with B (a scene batch's) [B, m, 3 | 4], B m <= 2^30.
    Returns (n or m, balls): balls is points itself when it has 4 columns, else a new [.., 4] tensor with r = +inf.
    ValueError for anything else."""
    import torch
    dims = 2 if B is None else 3
    shape = "[n, 3] or [n, 4]" if B is None else "[B, m, 3] or [B, m, 4]"
    if not isinstance(points, torch.Tensor) or points.dim() != dims or points.shape[-1] not in (3, 4):
        got = f"{points.dtype} {tuple(points.shape)}" if isinstance(points, torch.Tensor) else type(points).__name__
        raise ValueError(f"points must be a float32 CUDA tensor of shape {shape} (centre.xyz[, r]), got {got}")
    _check_tensor(device, "points", points, (torch.float32,), tuple(points.shape))
    count = int(points.shape[0]) if B is None else int(points.shape[1])
    if B is None and count > 1 << 30:
        raise ValueError(f"a nearest-sphere query takes at most 2^30 points, got {count}")
    if B is not None and int(points.shape[0]) != B:
        raise ValueError(f"points must have one row per scene of the batch ({B}), got {int(points.shape[0])}")
    if B is not None and B * count > 1 << 30:
        raise ValueError(f"a batch nearest-sphere query takes at most 2^30 points, got {B} x {count}")
    if points.shape[-1] == 4:
        return count, points
    return count, torch.cat([points, torch.full_like(points[..., :1], float("inf"))], -1)


def _camera7(cam7):
    """cam7 (look_from.xyz, look_at.xyz, fov) as a contiguous float32 [7] host array, from any host array-like of 7
    floating-point values; a CUDA tensor raises ValueError (reading it would synchronise the device), as does any other
    shape or dtype."""
    if type(cam7).__module__.startswith("torch"):
        if cam7.device.type != "cpu":
            raise ValueError(f"cam7 must be a host array of 7 floats, got a tensor on {cam7.device}")
        cam7 = cam7.numpy()
    a = np.asarray(cam7)
    if a.shape != (7,) or a.dtype.kind != "f":
        raise ValueError(f"cam7 must be a host array of 7 floats, got {a.dtype} {a.shape}")
    return np.ascontiguousarray(a, np.float32)


def camera_rays(camera, h, w, spp=1):
    """Camera rays of an h x w frame as render traces them: float32[h][w][spp][6] (origin, direction) of sample s of
    pixel (row j, column i), with the same float32 operations in the same order as the render kernels (ray.fut:109-114,
    150-154 and the spp extension of ray_b200.h).  camera: the 12 floats of PreparedScene.info()["camera"].  Through
    Context.trace_paths, quantised, these rays give the frame itself."""
    c = np.asarray(camera, np.float32).reshape(12)
    f = np.float32
    i = np.arange(w, dtype=np.float32)[None, :, None]
    hj = (f(h) - np.arange(h, dtype=np.float32))[:, None, None]   # f32(H - j): exact for any frame size render accepts
    if spp == 1:
        u = np.broadcast_to(i / f(w), (h, w, 1))
        v = np.broadcast_to(hj / f(h), (h, w, 1))
    else:
        off = host_sample_offsets(spp)
        u = np.broadcast_to((i + off[:, 0][None, None, :]) / f(w), (h, w, spp))
        v = np.broadcast_to((hj + off[:, 1][None, None, :]) / f(h), (h, w, spp))
    out = np.empty((h, w, spp, 6), np.float32)
    out[..., 0:3] = c[0:3]
    for a in range(3):   # llc + u*horizontal + v*vertical - origin, per component, left to right
        out[..., 3 + a] = ((c[3 + a] + u * c[6 + a]) + v * c[9 + a]) - c[a]
    return out


class _Handle:
    _free_fn = None

    def __init__(self, ctx, handle):
        self.ctx = ctx
        self.handle = handle

    def free(self):
        if self.handle and self.ctx.handle:
            getattr(self.ctx.lib, self._free_fn)(self.ctx.handle, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Scene(_Handle):
    """`scene` (ray.fut:171-174), opaque as in the generated API."""
    _free_fn = "futhark_free_opaque_scene"

    @property
    def num_spheres(self):
        return int(self.ctx.lib.ray_b200_scene_num_spheres(self.ctx.handle, self.handle))

    def arrays(self):
        n = self.num_spheres
        s = np.empty((n, 7), np.float32)
        c = np.empty(7, np.float32)
        self.ctx._check(self.ctx.lib.ray_b200_scene_get_arrays(self.ctx.handle, self.handle, _ptr(s), _ptr(c)))
        return s, c

    def store(self):
        p = C.c_void_p(None)
        n = C.c_size_t(0)
        self.ctx._check(self.ctx.lib.futhark_store_opaque_scene(self.ctx.handle, self.handle, C.byref(p), C.byref(n)))
        blob = C.string_at(p, n.value)
        _free(p)
        return blob


class PreparedScene(_Handle):
    """`prepared_scene` (ray.fut:239): LBVH + camera, resident in HBM."""
    _free_fn = "futhark_free_opaque_prepared_scene"

    def info(self):
        bi = BvhInfo()
        self.ctx._check(self.ctx.lib.ray_b200_prepared_info(self.ctx.handle, self.handle, C.byref(bi)))
        return {"n_leaves": bi.n_leaves, "n_inner": bi.n_inner, "max_depth": bi.max_depth,
                "refit_sweeps": bi.refit_sweeps, "stale_nodes": bi.stale_nodes, "smem_nodes": bi.smem_nodes,
                "root_box": np.array(bi.root_box[:], np.float32), "camera": np.array(bi.camera[:], np.float32)}

    def dump(self):
        n = int(self.info()["n_leaves"])
        out = dict(morton=np.empty(n, np.uint32), perm=np.empty(n, np.int32), left=np.empty(n - 1, np.int32),
                   right=np.empty(n - 1, np.int32), parent=np.empty(n - 1, np.int32),
                   boxes=np.empty((n - 1, 6), np.float32))
        self.ctx._check(self.ctx.lib.ray_b200_prepared_dump(self.ctx.handle, self.handle, _ptr(out["morton"]),
                                                            _ptr(out["perm"]), _ptr(out["left"]), _ptr(out["right"]),
                                                            _ptr(out["parent"]), _ptr(out["boxes"])))
        return out

    def packed(self):
        """The packed BVH2C arrays as they sit in HBM (nodes, nodes_soa, geom, colour)."""
        n = int(self.info()["n_leaves"])
        out = dict(nodes=np.empty((n - 1, 16), np.float32), nodes_soa=np.empty((4, n - 1, 4), np.float32),
                   geom=np.empty((n, 4), np.float32), colour=np.empty((n, 4), np.float32))
        self.ctx._check(self.ctx.lib.ray_b200_prepared_packed(self.ctx.handle, self.handle, _ptr(out["nodes"]),
                                                              _ptr(out["nodes_soa"]), _ptr(out["geom"]), _ptr(out["colour"])))
        return out

    def upload_bytes(self):
        return int(self.ctx.lib.ray_b200_prepared_upload_bytes(self.ctx.handle, self.handle))

    def device_bytes(self):
        return int(self.ctx.lib.ray_b200_prepared_device_bytes(self.ctx.handle, self.handle))

    def reupload(self):
        """Host->device copy of the packed BVH + spheres again (the H2D leg of bench.py's e2e step).  A scene last built
        from device memory is rebuilt from its own device arrays, with no copy."""
        self.ctx._check(self.ctx.lib.ray_b200_prepared_reupload(self.ctx.handle, self.handle))

    def update_from_ptr(self, spheres_dev, n, cam7=None):
        """ray_b200_prepared_update: replaces the scene's spheres by the n records at device address spheres_dev
        (float[n][7], read on the context's stream) and rebuilds its tree; cam7 (host [7]) replaces the camera, None keeps
        it.  Returns after the build's 32-byte read-back; spheres_dev may then be reused."""
        c = None if cam7 is None else _camera7(cam7)
        self.ctx._check(self.ctx.lib.ray_b200_prepared_update(self.ctx.handle, self.handle, _ptr(spheres_dev), int(n), _ptr(c)))

    def update(self, spheres, cam7=None):
        """Rebuilds the scene from spheres, a contiguous float32 CUDA tensor [n, 7] on the context's device (2 <= n <= 2^26;
        the layout of Context.scene_from_arrays), and cam7 (host [7]) or None to keep the camera.  The result is the scene
        prepare_scene makes from the same records, bit for bit; nothing is copied to or from the host.  Frames enqueued
        before the call render the old scene.  Waits for torch's current stream before the call."""
        import torch
        n = _sphere_rows(self.ctx.device, spheres)
        c = None if cam7 is None else _camera7(cam7)
        torch.cuda.current_stream(spheres.device).synchronize()   # spheres may still be in flight on torch's stream
        self.update_from_ptr(spheres.data_ptr(), n, c)

    def spheres(self):
        """(spheres, cam7): the scene's current records as a new CUDA float32 tensor [n, 7] in the order they were given,
        bit for bit, and its camera as a host float32 [7] array.  Synchronises the context."""
        import torch
        n = int(self.info()["n_leaves"])
        out = torch.empty((n, 7), dtype=torch.float32, device=torch.device("cuda", self.ctx.device))
        cam = np.empty(7, np.float32)
        torch.cuda.current_stream(out.device).synchronize()
        self.ctx._check(self.ctx.lib.ray_b200_prepared_spheres(self.ctx.handle, self.handle, _ptr(out.data_ptr()), _ptr(cam)))
        self.ctx.sync()
        return out, cam

    def store(self):
        p = C.c_void_p(None)
        n = C.c_size_t(0)
        self.ctx._check(self.ctx.lib.futhark_store_opaque_prepared_scene(self.ctx.handle, self.handle, C.byref(p), C.byref(n)))
        blob = C.string_at(p, n.value)
        _free(p)
        return blob


class SceneBatch(_Handle):
    """B scenes, of n spheres each or of counts[b] spheres (a ragged batch), built together from device memory, rendered
    in one launch and traced by ray queries in one launch (include/ray_b200.h "scene batches"; Context.render_scene_batch,
    Context.trace_scene_batch_*)."""
    _free_fn = "ray_b200_scene_batch_free"

    @property
    def shape(self):
        """(B, n), n = 0 when the members' counts differ"""
        b, n = C.c_int32(0), C.c_int64(0)
        self.ctx._check(self.ctx.lib.ray_b200_scene_batch_shape(self.ctx.handle, self.handle, C.byref(b), C.byref(n)))
        return int(b.value), int(n.value)

    @property
    def counts(self):
        """The B members' sphere counts, an int64 host array"""
        out = np.empty(self.shape[0], np.int64)
        self.ctx._check(self.ctx.lib.ray_b200_scene_batch_counts(self.ctx.handle, self.handle, out.ctypes.data))
        return out

    def update_from_ptr(self, spheres_dev, cams=None):
        """ray_b200_scene_batch_update: every member rebuilt from the records at device address spheres_dev (float[B][n][7],
        read on the context's stream) and the host cameras cams ([B, 7], None keeps them)."""
        c = None if cams is None else scene_batch_cameras(cams, self.shape[0])
        self.ctx._check(self.ctx.lib.ray_b200_scene_batch_update(self.ctx.handle, self.handle, _ptr(spheres_dev), _ptr(c)))

    def update_ragged_from_ptr(self, spheres_dev, counts, cams=None):
        """ray_b200_scene_batch_update_ragged: every member rebuilt from the records at device address spheres_dev
        (float[N][7], N = sum(counts), read on the context's stream), B new counts (host int64 array-like) and the host
        cameras cams ([B, 7], None keeps them)."""
        B = self.shape[0]
        c = np.ascontiguousarray(counts, np.int64)
        if c.shape != (B,):
            raise ValueError(f"counts must hold the batch's {B} counts, got shape {c.shape}")
        cam = None if cams is None else scene_batch_cameras(cams, B)
        self.ctx._check(self.ctx.lib.ray_b200_scene_batch_update_ragged(self.ctx.handle, self.handle, _ptr(spheres_dev),
                                                                        c.ctypes.data, _ptr(cam)))

    def update(self, spheres, cams=None, counts=None):
        """Rebuilds every member from spheres, a contiguous float32 CUDA tensor of the batch's shape [B, n, 7], and cams
        ([B, 7], see scene_batch_cameras) or None to keep the cameras.  With counts (B host integers, see
        scene_batch_counts; they may differ from the current ones), spheres is [sum(counts), 7], scene b's records from
        row counts[0] + .. + counts[b - 1].  Frames enqueued before the call render the old trees.  Waits for torch's
        current stream before the call."""
        import torch
        if counts is not None:
            B, c = scene_batch_counts(self.ctx.device, spheres, counts, B=self.shape[0])
            cam = None if cams is None else scene_batch_cameras(cams, B)
            torch.cuda.current_stream(spheres.device).synchronize()   # spheres may still be in flight on torch's stream
            self.update_ragged_from_ptr(spheres.data_ptr(), c, cam)
            return
        B, n = scene_batch_rows(self.ctx.device, spheres)
        if (B, n) != self.shape:
            raise ValueError(f"spheres must have the batch's shape {list(self.shape) + [7]}, got {list(spheres.shape)}")
        c = None if cams is None else scene_batch_cameras(cams, B)
        torch.cuda.current_stream(spheres.device).synchronize()   # spheres may still be in flight on torch's stream
        self.update_from_ptr(spheres.data_ptr(), c)

    def member(self, b):
        """Member b as a new, independent PreparedScene: bit for bit what Context.prepare_scene_device makes of its records."""
        out = C.c_void_p(None)
        self.ctx._check(self.ctx.lib.ray_b200_scene_batch_member(self.ctx.handle, self.handle, int(b), C.byref(out)))
        return PreparedScene(self.ctx, out.value)


class Image(_Handle):
    """`[h][w]i32` (ray.fut:164): packed 0x00RRGGBB, row 0 = top; lives on the device."""
    _free_fn = "futhark_free_i32_2d"

    @property
    def shape(self):
        s = self.ctx.lib.futhark_shape_i32_2d(self.ctx.handle, self.handle)
        return int(s[0]), int(s[1])

    def values(self, out=None):
        h, w = self.shape
        if out is None:
            out = np.empty((h, w), np.int32)
        self.ctx._check(self.ctx.lib.futhark_values_i32_2d(self.ctx.handle, self.handle, _ptr(out)))
        return out

    def device_ptr(self):
        return int(self.ctx.lib.futhark_values_raw_i32_2d(self.ctx.handle, self.handle) or 0)


class Context:
    """futhark_context + futhark_context_config (main.c:59-64)."""

    def __init__(self, device=None, kernel=None, spp=None, rank=None, world=None, **tuning):
        kid = KERNELS[kernel] if isinstance(kernel, str) else kernel
        self.lib = load_library("all" if kid in ALT_KERNELS else "")
        self.handle = None
        cfg = self.lib.futhark_context_config_new()
        if not cfg:
            raise RayError("futhark_context_config_new failed")
        try:
            if device is not None:
                self.lib.futhark_context_config_set_device(cfg, str(int(device)).encode())
            if kernel is not None:
                tuning["kernel"] = KERNELS[kernel] if isinstance(kernel, str) else int(kernel)
            if spp is not None:
                tuning["spp"] = int(spp)
            if rank is not None:
                tuning["rank"] = int(rank)
            if world is not None:
                tuning["world"] = int(world)
            for k, v in tuning.items():
                if self.lib.futhark_context_config_set_tuning_param(cfg, k.encode(), int(v)) != 0:
                    raise RayError(f"unknown tuning parameter {k!r}")
            h = self.lib.futhark_context_new(cfg)
        finally:
            self.lib.futhark_context_config_free(cfg)
        if not h:
            raise RayError("futhark_context_new returned NULL")
        self.handle = h
        err = self.get_error()
        if err is not None:  # main.c:64 asserts this is NULL
            self.lib.futhark_context_free(h)
            self.handle = None
            raise RayError(err)

    # -- errors --------------------------------------------------------------------------------
    def get_error(self):
        p = self.lib.futhark_context_get_error(self.handle)
        if not p:
            return None
        msg = C.string_at(p).decode(errors="replace")
        _free(p)
        return msg

    def _check(self, rc):
        if rc != 0:
            raise RayError(self.get_error() or f"ray_b200 call failed with code {rc}")

    def _out(self, cls, fn, *args):
        out = C.c_void_p(None)
        self._check(getattr(self.lib, fn)(self.handle, C.byref(out), *args))
        return cls(self, out.value)

    # -- the reference's entries ---------------------------------------------------------------
    def rgbbox(self):
        return self._out(Scene, "futhark_entry_rgbbox")

    def irreg(self):
        return self._out(Scene, "futhark_entry_irreg")

    def prepare_scene(self, h, w, scene):
        return self._out(PreparedScene, "futhark_entry_prepare_scene", int(h), int(w), scene.handle)

    def prepare_scene_device_from_ptr(self, h, w, spheres_dev, n, cam7):
        """ray_b200_prepare_scene_device: a prepared scene built from the n sphere records at device address spheres_dev
        (float[n][7], read on the context's stream) with the host camera cam7 ([7]).  Returns after the build's 32-byte
        read-back; spheres_dev may then be reused."""
        c = _camera7(cam7)
        return self._out(PreparedScene, "ray_b200_prepare_scene_device", int(h), int(w), _ptr(spheres_dev), int(n), _ptr(c))

    def prepare_scene_device(self, h, w, spheres, cam7):
        """prepare_scene from sphere records in device memory: spheres is a contiguous float32 CUDA tensor [n, 7] on the
        context's device (the layout of scene_from_arrays), cam7 a host array-like of 7 floats.  The prepared scene equals
        prepare_scene(h, w, scene_from_arrays(spheres, cam7)) bit for bit, and no record is copied to the host.  Waits for
        torch's current stream before the call; see PreparedScene.update for animating it."""
        import torch
        n = _sphere_rows(self.device, spheres)
        c = _camera7(cam7)
        torch.cuda.current_stream(spheres.device).synchronize()   # spheres may still be in flight on torch's stream
        return self.prepare_scene_device_from_ptr(h, w, spheres.data_ptr(), n, c)

    def prepare_scene_batch_from_ptr(self, h, w, spheres_dev, B, n, cams):
        """ray_b200_scene_batch_new_device: B scenes of n spheres from device address spheres_dev (float[B][n][7], read on
        the context's stream) with the host cameras cams ([B, 7]).  Returns after the build's one read-back."""
        c = scene_batch_cameras(cams, int(B))
        return self._out(SceneBatch, "ray_b200_scene_batch_new_device", int(h), int(w), _ptr(spheres_dev), int(B), int(n), _ptr(c))

    def prepare_scene_batch_ragged_from_ptr(self, h, w, spheres_dev, counts, cams):
        """ray_b200_scene_batch_new_ragged: B = len(counts) scenes of counts[b] spheres, back to back from device address
        spheres_dev (float[N][7], N = sum(counts), read on the context's stream) with the host cameras cams ([B, 7]).
        Returns after the build's one read-back."""
        c = np.ascontiguousarray(counts, np.int64)
        if c.ndim != 1:
            raise ValueError(f"counts must be a 1-d sequence of B integers, got shape {c.shape}")
        cam = scene_batch_cameras(cams, len(c))
        return self._out(SceneBatch, "ray_b200_scene_batch_new_ragged", int(h), int(w), _ptr(spheres_dev), len(c), c.ctypes.data,
                         _ptr(cam))

    def prepare_scene_batch(self, h, w, spheres, cams, counts=None):
        """A SceneBatch from spheres, a contiguous float32 CUDA tensor [B, n, 7] on the context's device (each scene in the
        layout of scene_from_arrays), and cams, [B, 7] cameras on the host or in a tensor.  Member b equals
        prepare_scene_device(h, w, spheres[b], cams[b]) bit for bit.  With counts (B host integers, see
        scene_batch_counts), the scenes may differ in size: spheres is [sum(counts), 7], scene b's records from row
        off_b = counts[0] + .. + counts[b - 1], and member b equals prepare_scene_device(h, w, spheres[off_b:off_b +
        counts[b]], cams[b]).  Waits for torch's current stream before the call."""
        import torch
        if counts is not None:
            B, c = scene_batch_counts(self.device, spheres, counts)
            if not scene_batch_frames_ok(B, int(h), int(w)):
                raise ValueError(f"{B} frames of {h}x{w} exceed one launch (2^25 tiles of 8x4 pixels, sides <= 65536)")
            cam = scene_batch_cameras(cams, B)
            torch.cuda.current_stream(spheres.device).synchronize()
            return self.prepare_scene_batch_ragged_from_ptr(h, w, spheres.data_ptr(), c, cam)
        B, n = scene_batch_rows(self.device, spheres)
        if not scene_batch_frames_ok(B, int(h), int(w)):
            raise ValueError(f"{B} frames of {h}x{w} exceed one launch (2^25 tiles of 8x4 pixels, sides <= 65536)")
        c = scene_batch_cameras(cams, B)
        torch.cuda.current_stream(spheres.device).synchronize()
        return self.prepare_scene_batch_from_ptr(h, w, spheres.data_ptr(), B, n, c)

    def render_scene_batch_into(self, batch, h, w, spp, out_pix_dev, out_rgb_dev=None):
        """One frame of every scene of a SceneBatch in one launch (ray_b200_render_scene_batch_into): out_pix_dev = device
        int32[B][h][w], out_rgb_dev = device float[B][h][w][3] or None.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_render_scene_batch_into(self.handle, batch.handle, int(h), int(w), int(spp),
                                                              _ptr(out_pix_dev), _ptr(out_rgb_dev)))

    def render_scene_batch(self, batch, h, w, spp=1, want_rgb=False):
        """Renders frame b of scene b for every member of a SceneBatch and returns CUDA int32 [B, h, w] pixels, and with
        want_rgb also the float32 [B, h, w, 3] framebuffers, as (pixels, rgb).  Frame b equals render_into of member b bit
        for bit.  Waits for torch's current stream before, and synchronises the context after the call."""
        import torch
        B = batch.shape[0]
        if not scene_batch_frames_ok(B, int(h), int(w)):
            raise ValueError(f"{B} frames of {h}x{w} exceed one launch (2^25 tiles of 8x4 pixels, sides <= 65536)")
        dev = torch.device("cuda", self.device)
        pix = torch.empty((B, int(h), int(w)), dtype=torch.int32, device=dev)
        rgb = torch.empty((B, int(h), int(w), 3), dtype=torch.float32, device=dev) if want_rgb else None
        torch.cuda.current_stream(dev).synchronize()
        self.render_scene_batch_into(batch, h, w, spp, pix.data_ptr(), rgb.data_ptr() if rgb is not None else None)
        self.sync()
        return (pix, rgb) if want_rgb else pix

    def render(self, h, w, prepared, spp=None):
        if spp is None:
            return self._out(Image, "futhark_entry_render", int(h), int(w), prepared.handle)
        return self._out(Image, "ray_b200_entry_render_spp", int(h), int(w), int(spp), prepared.handle)

    def sync(self):
        self._check(self.lib.futhark_context_sync(self.handle))

    def report(self):
        p = self.lib.futhark_context_report(self.handle)
        msg = C.string_at(p).decode()
        _free(p)
        return msg

    # -- extensions ----------------------------------------------------------------------------
    def scene(self, name, n=None, seed=1):
        if name == "rgbbox":
            return self.rgbbox()
        if name == "irreg":
            return self.irreg()
        if name == "random":
            return self.scene_random(n, seed)
        raise ValueError(f"unknown scene {name!r}")

    def scene_random(self, n, seed=1):
        return self._out(Scene, "ray_b200_scene_random", int(n), int(seed))

    def scene_from_arrays(self, spheres, cam7):
        s = np.ascontiguousarray(spheres, np.float32).reshape(-1, 7)
        c = np.ascontiguousarray(cam7, np.float32).reshape(7)
        return self._out(Scene, "ray_b200_scene_from_arrays", _ptr(s), s.shape[0], _ptr(c))

    def restore_scene(self, blob):
        h = self.lib.futhark_restore_opaque_scene(self.handle, blob)
        if not h:
            raise RayError(self.get_error() or "restore failed")
        return Scene(self, h)

    def restore_prepared_scene(self, blob):
        h = self.lib.futhark_restore_opaque_prepared_scene(self.handle, blob)
        if not h:
            raise RayError(self.get_error() or "restore failed")
        return PreparedScene(self, h)

    def set_stream(self, cuda_stream):
        """cuda_stream: a cudaStream_t handle (torch.cuda.Stream.cuda_stream).  torch's default stream has
        handle 0, which the C API reads as "restore the context's own stream"; it is passed as
        cudaStreamLegacy (0x1) instead so the work really lands on the default stream.  None restores."""
        if cuda_stream is None:
            h = None
        else:
            h = int(cuda_stream) or 1
        self._check(self.lib.ray_b200_context_set_stream(self.handle, C.c_void_p(h)))

    def set_spp(self, spp):
        self._check(self.lib.ray_b200_context_set_spp(self.handle, int(spp)))

    def set_kernel(self, kernel):
        self._check(self.lib.ray_b200_context_set_kernel(self.handle, KERNELS[kernel] if isinstance(kernel, str) else int(kernel)))

    def set_shard(self, rank, world):
        self._check(self.lib.ray_b200_context_set_shard(self.handle, int(rank), int(world)))

    @property
    def device(self):
        return int(self.lib.ray_b200_context_device(self.handle))

    def last_render_ms(self):
        ms = C.c_float(0)
        self._check(self.lib.ray_b200_context_last_render_ms(self.handle, C.byref(ms)))
        return float(ms.value)

    def trace_warps(self, enable=True):
        """Diagnostic: record when each warp of the warp-queue kernel runs out of work (see warp_trace)."""
        self._check(self.lib.ray_b200_context_trace_warps(self.handle, 1 if enable else 0))

    def warp_trace(self):
        """float32[SMs * warps]: exit time of every warp of the last traced render, in us after the first CTA started."""
        n = C.c_int64(0)
        self._check(self.lib.ray_b200_context_warp_trace(self.handle, None, 0, C.byref(n)))
        out = np.empty(n.value, np.float32)
        self._check(self.lib.ray_b200_context_warp_trace(self.handle, out.ctypes.data_as(C.POINTER(C.c_float)), n.value, C.byref(n)))
        return out

    def launch_count(self):
        return int(self.lib.ray_b200_context_launch_count(self.handle))

    def last_plan(self):
        """The plan of the last render kernel launch on this context (ray_b200_context_last_plan) as a dict of the fields
        of struct ray_b200_plan, with query as its name in QUERIES.  Host-only: call it after the launch's call returns."""
        p = Plan()
        self._check(self.lib.ray_b200_context_last_plan(self.handle, C.byref(p)))
        out = {k: int(getattr(p, k)) for k, _ in Plan._fields_}
        out["query"] = QUERIES[out["query"]]
        return out

    def render_into(self, out_pix_dev, h, w, prepared, spp=1, out_rgb_dev=None):
        self._check(self.lib.ray_b200_render_into(self.handle, _ptr(out_pix_dev), _ptr(out_rgb_dev), int(h), int(w), int(spp), prepared.handle))

    def render_accumulate_into(self, accum_dev, h, w, prepared, s_begin, s_end, out_pix_dev=None, out_rgb_dev=None):
        """Progressive rendering (ray_b200_render_accumulate): adds samples [s_begin, s_end) of every pixel to the running
        sums in accum_dev (device float[h][w][3]; not read when s_begin == 0), in sample order, and writes the frame at
        spp = s_end to out_pix_dev (device int32[h][w]) / out_rgb_dev (device float[h][w][3]) where given.  A chain of
        calls [0, a), [a, b), ... equals one render at the total spp, bit for bit.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_render_accumulate(self.handle, _ptr(accum_dev), int(h), int(w), int(s_begin), int(s_end),
                                                        _ptr(out_pix_dev), _ptr(out_rgb_dev), prepared.handle))

    def render_accumulate(self, prepared, accum, s_begin, s_end, want_rgb=False):
        """Adds samples [s_begin, s_end) of every pixel to accum, a contiguous float32 CUDA tensor [h, w, 3] on the
        context's device that holds the running sums of samples [0, s_begin) (not read when s_begin == 0), and returns
        the frame at spp = s_end: int32 [h, w] pixels, and with want_rgb also the float32 [h, w, 3] framebuffer, as
        (pixels, rgb).  With a shard set, the pixels of other ranks are 0.  Waits for torch's current stream before, and
        synchronises the context after the call."""
        import torch
        if not isinstance(accum, torch.Tensor) or accum.device.type != "cuda" or accum.device.index != self.device:
            raise ValueError(f"accum must be a CUDA tensor on cuda:{self.device}")
        if accum.dtype != torch.float32 or accum.dim() != 3 or accum.shape[2] != 3 or not accum.is_contiguous():
            raise ValueError(f"accum must be a contiguous float32 tensor of shape [h, w, 3], got {accum.dtype} {tuple(accum.shape)}")
        h, w = int(accum.shape[0]), int(accum.shape[1])
        pix = torch.zeros((h, w), dtype=torch.int32, device=accum.device)
        rgb = torch.zeros((h, w, 3), dtype=torch.float32, device=accum.device) if want_rgb else None
        # accum may still be in flight on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(accum.device).synchronize()
        self.render_accumulate_into(accum.data_ptr(), h, w, prepared, s_begin, s_end, pix.data_ptr(),
                                    rgb.data_ptr() if rgb is not None else None)
        self.sync()
        return (pix, rgb) if want_rgb else pix

    def render_adaptive_into(self, accum_dev, counts_dev, h, w, prepared, n_add, mask_dev=None, out_pix_dev=None,
                             out_rgb_dev=None):
        """Adaptive progressive rendering (ray_b200_render_adaptive): adds samples [c, c + n_add) to the running sum
        accum_dev[p] (device float[h][w][3]) of every pixel p that mask_dev (device uint8[h][w]; None = every pixel)
        selects, where c = counts_dev[p] (device int32[h][w]), raises the count by n_add and writes the pixel at
        spp = c + n_add to out_pix_dev (int32[h][w]) / out_rgb_dev (float[h][w][3]) where given.  Unselected pixels are
        neither read nor written.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_render_adaptive(self.handle, _ptr(accum_dev), _ptr(counts_dev), _ptr(mask_dev), int(h),
                                                      int(w), int(n_add), _ptr(out_pix_dev), _ptr(out_rgb_dev), prepared.handle))

    def render_adaptive_var_into(self, accum_dev, m2_dev, counts_dev, h, w, prepared, n_add, mask_dev=None, out_pix_dev=None,
                                 out_rgb_dev=None):
        """render_adaptive_into that also keeps each pixel's M2 (ray_b200_render_adaptive_var): m2_dev (device
        float[h][w][3]) is Welford's running sum of squared deviations of the pixel's samples, per channel, so that
        m2 / (count - 1) is their variance.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_render_adaptive_var(self.handle, _ptr(accum_dev), _ptr(m2_dev), _ptr(counts_dev),
                                                          _ptr(mask_dev), int(h), int(w), int(n_add), _ptr(out_pix_dev),
                                                          _ptr(out_rgb_dev), prepared.handle))

    def adaptive_select_into(self, accum_dev, m2_dev, counts_dev, h, w, rel_err, mean_floor, min_count, max_count, mask_dev,
                             n_selected_dev=None):
        """The pixels that still need samples (ray_b200_adaptive_select): mask_dev[p] (device uint8[h][w]) = 1 where
        0 <= count < max_count and either count < min_count or the pixel's variance of the mean, summed over the
        channels, is above (rel_err * (mean channel sum + mean_floor))^2; n_selected_dev (device int32, or None) gets
        the number of ones.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_adaptive_select(self.handle, _ptr(accum_dev), _ptr(m2_dev), _ptr(counts_dev), int(h),
                                                      int(w), float(rel_err), float(mean_floor), int(min_count),
                                                      int(max_count), _ptr(mask_dev), _ptr(n_selected_dev)))

    def render_adaptive(self, prepared, accum, counts, n_add, mask=None, pixels=None, rgb=None, m2=None):
        """Adds n_add samples to the pixels `mask` selects, each from its own count: accum is a float32 CUDA tensor
        [h, w, 3] of running sums, counts an int32 [h, w] tensor of how many samples each sum holds, mask a bool or uint8
        [h, w] tensor or None (every pixel); all contiguous and on the context's device.  accum and counts are updated in
        place.  pixels (int32 [h, w]) and rgb (float32 [h, w, 3]), where given, get the selected pixels at their new
        counts; the other pixels keep what they held.  m2 (float32 [h, w, 3]), where given, is each pixel's M2 and is
        updated too (ray_b200_render_adaptive_var; see adaptive_select).  Returns (pixels, rgb).  Waits for torch's
        current stream before, and synchronises the context after the call."""
        import torch
        check = lambda *a: _check_tensor(self.device, *a)
        if not isinstance(accum, torch.Tensor) or accum.dim() != 3:
            raise ValueError("accum must be a float32 CUDA tensor of shape [h, w, 3]")
        h, w = int(accum.shape[0]), int(accum.shape[1])
        check("accum", accum, (torch.float32,), (h, w, 3))
        if m2 is not None:
            check("m2", m2, (torch.float32,), (h, w, 3))
        check("counts", counts, (torch.int32,), (h, w))
        if mask is not None:
            check("mask", mask, (torch.bool, torch.uint8), (h, w))
        if pixels is not None:
            check("pixels", pixels, (torch.int32,), (h, w))
        if rgb is not None:
            check("rgb", rgb, (torch.float32,), (h, w, 3))
        # the tensors may still be in flight on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(accum.device).synchronize()
        ptr = lambda t: t.data_ptr() if t is not None else None
        if m2 is None:
            self.render_adaptive_into(accum.data_ptr(), counts.data_ptr(), h, w, prepared, n_add, ptr(mask), ptr(pixels), ptr(rgb))
        else:
            self.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, prepared, n_add, ptr(mask),
                                          ptr(pixels), ptr(rgb))
        self.sync()
        return pixels, rgb

    def adaptive_select(self, accum, m2, counts, rel_err, mean_floor, min_count, max_count, out=None):
        """The pixels of an adaptive frame that still need samples, by the noise estimate of render_adaptive(m2=...)
        (ray_b200_adaptive_select): accum and m2 are float32 CUDA tensors [h, w, 3], counts int32 [h, w], out a bool or
        uint8 [h, w] tensor or None (a new bool tensor); all contiguous and on the context's device.  A pixel with count n
        is selected when 0 <= n < max_count and either n < min_count or the variance of its mean, summed over the three
        channels, is above (rel_err * (mean channel sum + mean_floor))^2.  Returns (mask, n_selected), n_selected an int32
        CUDA tensor of shape [1].  Waits for torch's current stream before, and synchronises the context after the call."""
        import torch
        check = lambda *a: _check_tensor(self.device, *a)
        if not isinstance(accum, torch.Tensor) or accum.dim() != 3:
            raise ValueError("accum must be a float32 CUDA tensor of shape [h, w, 3]")
        h, w = int(accum.shape[0]), int(accum.shape[1])
        check("accum", accum, (torch.float32,), (h, w, 3))
        check("m2", m2, (torch.float32,), (h, w, 3))
        check("counts", counts, (torch.int32,), (h, w))
        if out is None:
            out = torch.empty((h, w), dtype=torch.bool, device=accum.device)
        check("out", out, (torch.bool, torch.uint8), (h, w))
        n_sel = torch.empty(1, dtype=torch.int32, device=accum.device)
        torch.cuda.current_stream(accum.device).synchronize()
        self.adaptive_select_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, rel_err, mean_floor, min_count,
                                  max_count, out.data_ptr(), n_sel.data_ptr())
        self.sync()
        return out, n_sel

    def render_converged(self, prepared, h, w, rel_err, mean_floor=0.1, min_spp=8, step=8, max_spp=512, want_rgb=False):
        """Renders the prepared scene at h x w until every pixel's noise estimate is within rel_err, at most max_spp
        samples per pixel: min_spp samples everywhere, then rounds of `step` more samples for the pixels adaptive_select
        still selects (min_count = min_spp, max_count = max_spp - step + 1, so no pixel passes max_spp), until a round
        selects none.  A pixel's target is rel_err times (its mean channel sum + mean_floor).  The floor keeps dark
        pixels from asking for a relative error of a mean near 0, which no sample count reaches; the default 0.1 is a
        channel sum of about 8 / 255 per channel, the darkest level the quantised pixel shows apart from black.
        Every pixel equals render_into(spp = counts[p]) at its own count.  Reads the selected count once per round.
        Returns (pixels int32 [h, w], rgb float32 [h, w, 3] if want_rgb, counts int32 [h, w],
        {"rounds": calls of the render kernel, "samples": samples traced}).  Waits for torch's current stream before,
        and synchronises the context after the call."""
        import torch
        if min_spp < 2 or step < 1 or max_spp < min_spp:
            raise ValueError(f"render_converged: need min_spp >= 2, step >= 1 and max_spp >= min_spp, got {min_spp}, {step}, {max_spp}")
        dev = torch.device("cuda", self.device)
        accum = torch.empty((h, w, 3), dtype=torch.float32, device=dev)
        m2 = torch.empty((h, w, 3), dtype=torch.float32, device=dev)
        counts = torch.zeros((h, w), dtype=torch.int32, device=dev)
        pix = torch.zeros((h, w), dtype=torch.int32, device=dev)
        rgb = torch.zeros((h, w, 3), dtype=torch.float32, device=dev) if want_rgb else None
        mask = torch.empty((h, w), dtype=torch.bool, device=dev)
        n_sel = torch.empty(1, dtype=torch.int32, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        ptr = lambda t: t.data_ptr() if t is not None else None
        self.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, prepared, min_spp, None,
                                      pix.data_ptr(), ptr(rgb))
        rounds, samples = 1, h * w * min_spp
        while min_spp + step <= max_spp:
            self.adaptive_select_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, rel_err, mean_floor, min_spp,
                                      max_spp - step + 1, mask.data_ptr(), n_sel.data_ptr())
            self.render_adaptive_var_into(accum.data_ptr(), m2.data_ptr(), counts.data_ptr(), h, w, prepared, step,
                                          mask.data_ptr(), pix.data_ptr(), ptr(rgb))
            self.sync()
            n = int(n_sel.item())
            if n == 0:
                break
            rounds += 1
            samples += n * step
        self.sync()
        stats = {"rounds": rounds, "samples": samples}
        return (pix, rgb, counts, stats) if want_rgb else (pix, counts, stats)

    def render_views_into(self, prepared, cams, h, w, spp, out_pix_dev, out_rgb_dev=None):
        """Several views of one prepared scene in one launch (ray_b200_render_views_into): cams = host [V, 7] cameras
        (look_from.xyz, look_at.xyz, fov; see camera_table), out_pix_dev = device int32[V][h][w], out_rgb_dev = device
        float[V][h][w][3] or None.  View v equals render_into of a scene prepared at (h, w) with camera cams[v], bit for
        bit.  Asynchronous on the context's stream; cams may be reused once the call returns."""
        c = camera_table(cams)
        self._check(self.lib.ray_b200_render_views_into(self.handle, prepared.handle, _ptr(c), c.shape[0], int(h), int(w),
                                                        int(spp), _ptr(out_pix_dev), _ptr(out_rgb_dev)))

    def render_views(self, prepared, cams, h, w, spp=1, want_rgb=False):
        """Renders V views of one prepared scene (cams: host [V, 7], see camera_table) and returns CUDA int32 [V, h, w]
        pixels, and with want_rgb also the float32 [V, h, w, 3] framebuffers, as (pixels, rgb).  Waits for torch's current
        stream before, and synchronises the context after the call."""
        import torch
        c = camera_table(cams)
        dev = torch.device("cuda", self.device)
        pix = torch.empty((c.shape[0], int(h), int(w)), dtype=torch.int32, device=dev)
        rgb = torch.empty((c.shape[0], int(h), int(w), 3), dtype=torch.float32, device=dev) if want_rgb else None
        # the outputs' memory may still be in use on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(dev).synchronize()
        self.render_views_into(prepared, c, h, w, spp, pix.data_ptr(), rgb.data_ptr() if rgb is not None else None)
        self.sync()
        return (pix, rgb) if want_rgb else pix

    GBUFFER_OUTPUTS = ("id", "depth", "normal", "albedo", "coverage")

    def render_gbuffer_into(self, prepared, h, w, spp, id_dev=0, depth_dev=0, normal_dev=0, albedo_dev=0, coverage_dev=0):
        """The first-hit buffers of an h x w frame at spp samples (ray_b200_render_gbuffer), written to the device buffers
        given (0 / None = not written): id_dev int32[h][w] (sphere of sample 0's first hit, -1 = none), depth_dev
        float[h][w] (its t along the camera ray, -1 = none), normal_dev and albedo_dev float[h][w][3] (the mean first-hit
        normal, and the mean of the hit sphere's colour or the sky's), coverage_dev int32[h][w] (samples that hit).
        Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_render_gbuffer(self.handle, prepared.handle, int(h), int(w), int(spp), _ptr(id_dev),
                                                     _ptr(depth_dev), _ptr(normal_dev), _ptr(albedo_dev), _ptr(coverage_dev)))

    def render_gbuffer(self, prepared, h, w, spp=1, outputs=GBUFFER_OUTPUTS):
        """The first-hit buffers of the prepared scene at h x w and spp samples per pixel, as a dict of new CUDA tensors
        on the context's device, one per name in `outputs`: "id" int32 [h, w], "depth" float32 [h, w], "normal" and
        "albedo" float32 [h, w, 3], "coverage" int32 [h, w] (see render_gbuffer_into and ray_b200_render_gbuffer for the
        rule).  Waits for torch's current stream before, and synchronises the context after the call."""
        import torch
        names = tuple(outputs)
        for n in names:
            if n not in self.GBUFFER_OUTPUTS:
                raise ValueError(f"render_gbuffer: unknown output {n!r}; the outputs are {', '.join(self.GBUFFER_OUTPUTS)}")
        if not names:
            raise ValueError("render_gbuffer: no output requested")
        dev = torch.device("cuda", self.device)
        h, w = int(h), int(w)
        shape = {"id": ((h, w), torch.int32), "depth": ((h, w), torch.float32), "normal": ((h, w, 3), torch.float32),
                 "albedo": ((h, w, 3), torch.float32), "coverage": ((h, w), torch.int32)}
        out = {n: torch.empty(shape[n][0], dtype=shape[n][1], device=dev) for n in self.GBUFFER_OUTPUTS if n in names}
        # the outputs' memory may still be in use on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(dev).synchronize()
        ptr = lambda n: out[n].data_ptr() if n in out else 0
        self.render_gbuffer_into(prepared, h, w, spp, ptr("id"), ptr("depth"), ptr("normal"), ptr("albedo"), ptr("coverage"))
        self.sync()
        return out

    def render_host(self, h, w, prepared, spp=1, want_rgb=False, out=None):
        pix = out if out is not None else np.empty((h, w), np.int32)
        rgb = np.empty((h, w, 3), np.float32) if want_rgb else None
        self._check(self.lib.ray_b200_render_host(self.handle, _ptr(pix), _ptr(rgb), int(h), int(w), int(spp), prepared.handle))
        return (pix, rgb) if want_rgb else pix

    def shard_tiles(self, h, w, rank, world):
        return int(self.lib.ray_b200_shard_tiles(int(h), int(w), int(rank), int(world)))

    def shard_tiles_padded(self, h, w, world):
        return int(self.lib.ray_b200_shard_tiles_padded(int(h), int(w), int(world)))

    def render_shard_into(self, out_tiles_dev, h, w, prepared, spp=1):
        self._check(self.lib.ray_b200_render_shard_into(self.handle, _ptr(out_tiles_dev), int(h), int(w), int(spp), prepared.handle))

    def render_batch(self, jobs):
        """jobs: sequence of dicts(prepared=, h=, w=, out_dev=, spp=0, shard_layout=False, out_rgb_dev=None).  Enqueues all
        frames as one stream-ordered operation with up to two of them in flight (ray_b200_render_batch)."""
        arr = (RenderJob * len(jobs))()
        for a, j in zip(arr, jobs):
            a.prepared = j["prepared"].handle
            a.h, a.w = int(j["h"]), int(j["w"])
            a.spp = int(j.get("spp") or 0)
            a.shard_layout = 1 if j.get("shard_layout") else 0
            a.out_dev = int(j["out_dev"])
            a.out_rgb_dev = int(j["out_rgb_dev"]) if j.get("out_rgb_dev") is not None else None
            a.wait_flag = int(j["wait_flag"]) if j.get("wait_flag") else None   # peer-frame protocol (ray_b200.h)
            a.wait_value = int(j.get("wait_value") or 0)
            a.done_flag = int(j["done_flag"]) if j.get("done_flag") else None
        self._check(self.lib.ray_b200_render_batch(self.handle, arr, len(jobs)))

    def set_pipeline(self, on=True):
        """Pipelined submission: render_batch stops joining its second lane (frames of consecutive calls overlap)."""
        self._check(self.lib.ray_b200_context_set_pipeline(self.handle, 1 if on else 0))

    def pipeline_join(self):
        self._check(self.lib.ray_b200_pipeline_join(self.handle))

    # -- peer-memory frames (include/ray_b200.h): raw device addresses as ints ---------------------------------
    def ipc_alloc(self, nbytes):
        """cudaMalloc'ed, zeroed device memory + its 64-byte CUDA IPC handle: (address, handle bytes)."""
        ptr = C.c_void_p(None)
        handle = (C.c_ubyte * 64)()
        self._check(self.lib.ray_b200_ipc_alloc(self.handle, int(nbytes), C.byref(ptr), handle))
        return int(ptr.value), bytes(handle)

    def ipc_free(self, ptr):
        self._check(self.lib.ray_b200_ipc_free(self.handle, C.c_void_p(int(ptr))))

    def ipc_open(self, handle):
        """Maps another process's ipc_alloc allocation (a peer GPU's memory over NVLink); returns the local address."""
        ptr = C.c_void_p(None)
        buf = (C.c_ubyte * 64).from_buffer_copy(bytes(handle))
        self._check(self.lib.ray_b200_ipc_open(self.handle, buf, C.byref(ptr)))
        return int(ptr.value)

    def ipc_close(self, ptr):
        self._check(self.lib.ray_b200_ipc_close(self.handle, C.c_void_p(int(ptr))))

    def flag_wait(self, flag_ptr, value, stream=None, timeout_ms=5000):
        self._check(self.lib.ray_b200_flag_wait(self.handle, C.c_void_p(int(stream) if stream else None), C.c_void_p(int(flag_ptr)),
                                                int(value) & 0xffffffff, int(timeout_ms)))

    def flag_set(self, flag_ptr, value, stream=None):
        self._check(self.lib.ray_b200_flag_set(self.handle, C.c_void_p(int(stream) if stream else None), C.c_void_p(int(flag_ptr)),
                                               int(value) & 0xffffffff))

    def flag_timeouts(self):
        n = C.c_int64(0)
        self._check(self.lib.ray_b200_flag_status(self.handle, C.byref(n)))
        return int(n.value)

    def copy_to_host_async(self, host_ptr, dev_ptr, nbytes, stream=None):
        self._check(self.lib.ray_b200_copy_to_host_async(self.handle, C.c_void_p(int(stream) if stream else None), C.c_void_p(int(host_ptr)),
                                                         C.c_void_p(int(dev_ptr)), int(nbytes)))

    def detile(self, gathered_dev, out_pix_dev, h, w, world):
        self._check(self.lib.ray_b200_detile(self.handle, _ptr(gathered_dev), _ptr(out_pix_dev), int(h), int(w), int(world)))

    # -- ray queries (include/ray_b200.h): caller-supplied rays against a prepared scene --------------------------
    def trace_hits_into(self, rays_dev, n, prepared, hits_dev, t_min=0.0, t_max=1e9):
        """Closest hit (objs_hit, ray.fut:76-86) of n rays: rays_dev = device float[n][6] (origin, direction), hits_dev =
        device Hit[n].  Asynchronous on the context's stream, like render_into."""
        self._check(self.lib.ray_b200_trace_hits(self.handle, prepared.handle, _ptr(rays_dev), int(n), float(t_min), float(t_max),
                                                 _ptr(hits_dev)))

    def trace_paths_into(self, rays_dev, n, prepared, rgb_dev, segments_dev=None, max_depth=50):
        """Colour (ray_colour, ray.fut:126-148) of n rays into device float[n][3], and optionally the objs_hit calls of
        every path into device int32[n].  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_trace_paths(self.handle, prepared.handle, _ptr(rays_dev), int(n), int(max_depth),
                                                  _ptr(rgb_dev), _ptr(segments_dev)))

    def trace_occluded_into(self, rays_dev, n, prepared, out_dev, t_min=0.0, t_max=1e9):
        """Occlusion of n rays: out_dev = device uint8[n] (a torch.bool buffer), 1 where some sphere the BVH walk reaches
        is hit in (t_min, t_max), else 0.  For point-to-point visibility pass direction = target - origin and an interval
        such as (1e-4, 1 - 1e-4).  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_trace_occluded(self.handle, prepared.handle, _ptr(rays_dev), int(n), float(t_min),
                                                     float(t_max), _ptr(out_dev)))

    def trace_multi_hits_into(self, rays_dev, n, prepared, k, hits_dev, counts_dev=None, t_min=0.0, t_max=1e9):
        """The k nearest sphere intersections of n rays in (t_min, t_max): hits_dev = device Hit[n][k], in ascending t
        (then Morton-sorted leaf), empty records (t = -1, sphere = -1) after the last; counts_dev = device int32[n]
        (or None) = every sphere the BVH walk reaches that is hit in the interval, not capped at k.  No epsilon, one
        record per sphere.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_trace_multi_hits(self.handle, prepared.handle, _ptr(rays_dev), int(n), float(t_min),
                                                       float(t_max), int(k), _ptr(hits_dev), _ptr(counts_dev)))

    def trace_hits_ranged_into(self, rays_dev, n, prepared, hits_dev):
        """trace_hits_into for rays that carry their own interval: rays_dev = device Ray[n] (float[n][8]: origin, t_min,
        direction, t_max), 4-byte aligned.  A ray whose interval the per-call form would reject (t_min not finite and
        >= 0, t_max not finite) gets the empty record.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_trace_hits_ranged(self.handle, prepared.handle, _ptr(rays_dev), int(n), _ptr(hits_dev)))

    def trace_occluded_ranged_into(self, rays_dev, n, prepared, out_dev):
        """trace_occluded_into for rays that carry their own interval (device Ray[n]); an invalid interval gives 0."""
        self._check(self.lib.ray_b200_trace_occluded_ranged(self.handle, prepared.handle, _ptr(rays_dev), int(n), _ptr(out_dev)))

    def trace_multi_hits_ranged_into(self, rays_dev, n, prepared, k, hits_dev, counts_dev=None):
        """trace_multi_hits_into for rays that carry their own interval (device Ray[n]); an invalid interval gives k
        empty records and a count of 0."""
        self._check(self.lib.ray_b200_trace_multi_hits_ranged(self.handle, prepared.handle, _ptr(rays_dev), int(n), int(k),
                                                              _ptr(hits_dev), _ptr(counts_dev)))

    def _rays_tensor(self, rays, ranged_ok=False, t_min=None, t_max=None):
        """Checks a tensor of rays: [n, 6] (origin, direction) or, where ranged_ok, [n, 8] (Ray: origin, t_min,
        direction, t_max), which carries its own interval and so takes no t_min= / t_max=.  Returns (torch, ranged)."""
        import torch
        widths = (6, 8) if ranged_ok else (6,)
        shapes = " or ".join(f"[n, {w}]" for w in widths)
        if isinstance(rays, torch.Tensor) and (rays.dim() != 2 or rays.shape[1] not in widths):
            raise ValueError(f"rays must be a contiguous float32 tensor of shape {shapes}, got {rays.dtype} {tuple(rays.shape)}")
        ranged = isinstance(rays, torch.Tensor) and rays.shape[1] == 8
        if ranged and (t_min is not None or t_max is not None):
            raise ValueError("rays of shape [n, 8] carry their own (t_min, t_max): pass t_min= / t_max= only with [n, 6] rays")
        if not isinstance(rays, torch.Tensor) or rays.device.type != "cuda" or rays.device.index != self.device:
            raise ValueError(f"rays must be a CUDA tensor on cuda:{self.device}")
        if rays.dtype != torch.float32 or not rays.is_contiguous():
            raise ValueError(f"rays must be a contiguous float32 tensor of shape {shapes}, got {rays.dtype} {tuple(rays.shape)}")
        # the rays may still be in flight on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(rays.device).synchronize()
        return torch, ranged

    def trace_hits(self, prepared, rays, t_min=None, t_max=None):
        """Closest hits of a [n, 6] float32 CUDA tensor of rays in (t_min, t_max) (default (0, 1e9)), or of a [n, 8] one
        whose rays carry their own interval (Ray; no t_min= / t_max= then).  Returns dict(t [n], sphere [n] int32,
        p [n, 3], normal [n, 3]): views of one [n, 8] buffer of Hit records.  t = -1 and sphere = -1 where a ray hits
        nothing.  Waits for torch's current stream before, and synchronises the context after the query."""
        torch, ranged = self._rays_tensor(rays, True, t_min, t_max)
        n = rays.shape[0]
        buf = torch.empty((n, 8), dtype=torch.float32, device=rays.device)
        if ranged:
            self.trace_hits_ranged_into(rays.data_ptr(), n, prepared, buf.data_ptr())
        else:
            self.trace_hits_into(rays.data_ptr(), n, prepared, buf.data_ptr(), t_min=_or(t_min, 0.0), t_max=_or(t_max, 1e9))
        self.sync()
        return {"t": buf[:, 0], "sphere": buf[:, 1].view(torch.int32), "p": buf[:, 2:5], "normal": buf[:, 5:8]}

    def trace_paths(self, prepared, rays, max_depth=50):
        """Colours of a [n, 6] float32 CUDA tensor of rays: (rgb [n, 3] float32, segments [n] int32 = objs_hit calls of
        every path).  Waits for torch's current stream before, and synchronises the context after the query."""
        torch, _ = self._rays_tensor(rays)
        n = rays.shape[0]
        rgb = torch.empty((n, 3), dtype=torch.float32, device=rays.device)
        seg = torch.empty((n,), dtype=torch.int32, device=rays.device)
        self.trace_paths_into(rays.data_ptr(), n, prepared, rgb.data_ptr(), seg.data_ptr(), max_depth=max_depth)
        self.sync()
        return rgb, seg

    def trace_occluded(self, prepared, rays, t_min=None, t_max=None):
        """Occlusion of a [n, 6] float32 CUDA tensor of rays in (t_min, t_max) (default (0, 1e9)), or of a [n, 8] one
        whose rays carry their own interval: torch.bool [n].  Waits for torch's current stream before, and synchronises
        the context after the query."""
        torch, ranged = self._rays_tensor(rays, True, t_min, t_max)
        n = rays.shape[0]
        out = torch.empty((n,), dtype=torch.bool, device=rays.device)
        if ranged:
            self.trace_occluded_ranged_into(rays.data_ptr(), n, prepared, out.data_ptr())
        else:
            self.trace_occluded_into(rays.data_ptr(), n, prepared, out.data_ptr(), t_min=_or(t_min, 0.0), t_max=_or(t_max, 1e9))
        self.sync()
        return out

    def trace_multi_hits(self, prepared, rays, k, t_min=None, t_max=None):
        """The k nearest sphere intersections of a [n, 6] float32 CUDA tensor of rays in (t_min, t_max) (default
        (0, 1e9)), or of a [n, 8] one whose rays carry their own interval.  Returns dict(t [n, k], sphere [n, k] int32,
        p [n, k, 3], normal [n, k, 3], count [n] int32): the first four are views of one [n, k, 8] buffer of Hit records.
        Waits for torch's current stream before, and synchronises the context after the query."""
        torch, ranged = self._rays_tensor(rays, True, t_min, t_max)
        n = rays.shape[0]
        buf = torch.empty((n, int(k), 8), dtype=torch.float32, device=rays.device)
        count = torch.empty((n,), dtype=torch.int32, device=rays.device)
        if ranged:
            self.trace_multi_hits_ranged_into(rays.data_ptr(), n, prepared, k, buf.data_ptr(), count.data_ptr())
        else:
            self.trace_multi_hits_into(rays.data_ptr(), n, prepared, k, buf.data_ptr(), count.data_ptr(), t_min=_or(t_min, 0.0),
                                       t_max=_or(t_max, 1e9))
        self.sync()
        return {"t": buf[..., 0], "sphere": buf[..., 1].view(torch.int32), "p": buf[..., 2:5], "normal": buf[..., 5:8],
                "count": count}

    # -- ray queries of a scene batch (include/ray_b200.h "scene batches"): m rays per scene, all B scenes in one launch
    def trace_scene_batch_hits_into(self, rays_dev, m, batch, hits_dev, t_min=0.0, t_max=1e9):
        """trace_hits_into for every scene of a SceneBatch: rays_dev = device float[B][m][6], ray j of scene b at b m + j,
        hits_dev = device Hit[B][m]; sphere is the index into the ray's own scene's records.  One launch, asynchronous on
        the context's stream."""
        self._check(self.lib.ray_b200_scene_batch_trace_hits(self.handle, batch.handle, _ptr(rays_dev), int(m), float(t_min),
                                                             float(t_max), _ptr(hits_dev)))

    def trace_scene_batch_paths_into(self, rays_dev, m, batch, rgb_dev, segments_dev=None, max_depth=50):
        """trace_paths_into for every scene of a SceneBatch: rgb_dev = device float[B][m][3], segments_dev = device
        int32[B][m] or None."""
        self._check(self.lib.ray_b200_scene_batch_trace_paths(self.handle, batch.handle, _ptr(rays_dev), int(m), int(max_depth),
                                                              _ptr(rgb_dev), _ptr(segments_dev)))

    def trace_scene_batch_occluded_into(self, rays_dev, m, batch, out_dev, t_min=0.0, t_max=1e9):
        """trace_occluded_into for every scene of a SceneBatch: out_dev = device uint8[B][m]."""
        self._check(self.lib.ray_b200_scene_batch_trace_occluded(self.handle, batch.handle, _ptr(rays_dev), int(m), float(t_min),
                                                                 float(t_max), _ptr(out_dev)))

    def trace_scene_batch_multi_hits_into(self, rays_dev, m, batch, k, hits_dev, counts_dev=None, t_min=0.0, t_max=1e9):
        """trace_multi_hits_into for every scene of a SceneBatch: hits_dev = device Hit[B][m][k], counts_dev = device
        int32[B][m] or None."""
        self._check(self.lib.ray_b200_scene_batch_trace_multi_hits(self.handle, batch.handle, _ptr(rays_dev), int(m), float(t_min),
                                                                   float(t_max), int(k), _ptr(hits_dev), _ptr(counts_dev)))

    def trace_scene_batch_hits_ranged_into(self, rays_dev, m, batch, hits_dev):
        """trace_scene_batch_hits_into for rays that carry their own interval: rays_dev = device Ray[B][m]."""
        self._check(self.lib.ray_b200_scene_batch_trace_hits_ranged(self.handle, batch.handle, _ptr(rays_dev), int(m), _ptr(hits_dev)))

    def trace_scene_batch_occluded_ranged_into(self, rays_dev, m, batch, out_dev):
        """trace_scene_batch_occluded_into for rays that carry their own interval (device Ray[B][m])."""
        self._check(self.lib.ray_b200_scene_batch_trace_occluded_ranged(self.handle, batch.handle, _ptr(rays_dev), int(m),
                                                                        _ptr(out_dev)))

    def trace_scene_batch_multi_hits_ranged_into(self, rays_dev, m, batch, k, hits_dev, counts_dev=None):
        """trace_scene_batch_multi_hits_into for rays that carry their own interval (device Ray[B][m])."""
        self._check(self.lib.ray_b200_scene_batch_trace_multi_hits_ranged(self.handle, batch.handle, _ptr(rays_dev), int(m), int(k),
                                                                          _ptr(hits_dev), _ptr(counts_dev)))

    def _batch_rays_tensor(self, batch, rays, ranged_ok=False, t_min=None, t_max=None):
        """Checks a tensor of rays of a scene batch: [B, m, 6] or, where ranged_ok, [B, m, 8] (Ray), with B the batch's
        own, m rays per scene and B m <= 2^30; [B, m, 8] rays take no t_min= / t_max=.  Returns (torch, ranged, m)."""
        import torch
        widths = (6, 8) if ranged_ok else (6,)
        shapes = " or ".join(f"[B, m, {w}]" for w in widths)
        if isinstance(rays, torch.Tensor) and (rays.dim() != 3 or rays.shape[2] not in widths):
            raise ValueError(f"rays must be a contiguous float32 tensor of shape {shapes}, got {rays.dtype} {tuple(rays.shape)}")
        ranged = isinstance(rays, torch.Tensor) and rays.shape[2] == 8
        if ranged and (t_min is not None or t_max is not None):
            raise ValueError("rays of shape [B, m, 8] carry their own (t_min, t_max): pass t_min= / t_max= only with [B, m, 6] rays")
        if not isinstance(rays, torch.Tensor) or rays.device.type != "cuda" or rays.device.index != self.device:
            raise ValueError(f"rays must be a CUDA tensor on cuda:{self.device}")
        if rays.dtype != torch.float32 or not rays.is_contiguous():
            raise ValueError(f"rays must be a contiguous float32 tensor of shape {shapes}, got {rays.dtype} {tuple(rays.shape)}")
        B, m = int(rays.shape[0]), int(rays.shape[1])
        if B != batch.shape[0]:
            raise ValueError(f"rays must have one row per scene of the batch ({batch.shape[0]}), got {B}")
        if B * m > 1 << 30:
            raise ValueError(f"a batch query traces at most 2^30 rays, got {B} x {m}")
        # the rays may still be in flight on torch's stream, which the context's own stream is not ordered after
        torch.cuda.current_stream(rays.device).synchronize()
        return torch, ranged, m

    def trace_scene_batch_hits(self, batch, rays, t_min=None, t_max=None):
        """Closest hits in every scene of a SceneBatch: rays is a [B, m, 6] float32 CUDA tensor, m rays per scene, traced in
        (t_min, t_max) (default (0, 1e9)), or a [B, m, 8] one whose rays carry their own interval (Ray).  Returns dict(t
        [B, m], sphere [B, m] int32, p [B, m, 3], normal [B, m, 3]) as trace_hits does, sphere indexing the ray's own
        scene's records.  Waits for torch's current stream before, and synchronises the context after the query."""
        torch, ranged, m = self._batch_rays_tensor(batch, rays, True, t_min, t_max)
        buf = torch.empty((rays.shape[0], m, 8), dtype=torch.float32, device=rays.device)
        if ranged:
            self.trace_scene_batch_hits_ranged_into(rays.data_ptr(), m, batch, buf.data_ptr())
        else:
            self.trace_scene_batch_hits_into(rays.data_ptr(), m, batch, buf.data_ptr(), t_min=_or(t_min, 0.0), t_max=_or(t_max, 1e9))
        self.sync()
        return {"t": buf[..., 0], "sphere": buf[..., 1].view(torch.int32), "p": buf[..., 2:5], "normal": buf[..., 5:8]}

    def trace_scene_batch_paths(self, batch, rays, max_depth=50):
        """Colours of a [B, m, 6] float32 CUDA tensor of rays, each in its own scene of a SceneBatch: (rgb [B, m, 3]
        float32, segments [B, m] int32).  Waits for torch's current stream before, and synchronises the context after."""
        torch, _, m = self._batch_rays_tensor(batch, rays)
        B = rays.shape[0]
        rgb = torch.empty((B, m, 3), dtype=torch.float32, device=rays.device)
        seg = torch.empty((B, m), dtype=torch.int32, device=rays.device)
        self.trace_scene_batch_paths_into(rays.data_ptr(), m, batch, rgb.data_ptr(), seg.data_ptr(), max_depth=max_depth)
        self.sync()
        return rgb, seg

    def trace_scene_batch_occluded(self, batch, rays, t_min=None, t_max=None):
        """Occlusion in every scene of a SceneBatch of [B, m, 6] rays in (t_min, t_max) (default (0, 1e9)), or of [B, m, 8]
        rays with their own intervals: torch.bool [B, m].  Waits for torch's current stream before, and synchronises the
        context after the query."""
        torch, ranged, m = self._batch_rays_tensor(batch, rays, True, t_min, t_max)
        out = torch.empty((rays.shape[0], m), dtype=torch.bool, device=rays.device)
        if ranged:
            self.trace_scene_batch_occluded_ranged_into(rays.data_ptr(), m, batch, out.data_ptr())
        else:
            self.trace_scene_batch_occluded_into(rays.data_ptr(), m, batch, out.data_ptr(), t_min=_or(t_min, 0.0),
                                                 t_max=_or(t_max, 1e9))
        self.sync()
        return out

    def trace_scene_batch_multi_hits(self, batch, rays, k, t_min=None, t_max=None):
        """The k nearest sphere intersections in every scene of a SceneBatch of [B, m, 6] rays in (t_min, t_max) (default
        (0, 1e9)), or of [B, m, 8] rays with their own intervals.  Returns dict(t [B, m, k], sphere [B, m, k] int32,
        p [B, m, k, 3], normal [B, m, k, 3], count [B, m] int32).  Waits for torch's current stream before, and
        synchronises the context after the query."""
        torch, ranged, m = self._batch_rays_tensor(batch, rays, True, t_min, t_max)
        B = rays.shape[0]
        buf = torch.empty((B, m, int(k), 8), dtype=torch.float32, device=rays.device)
        count = torch.empty((B, m), dtype=torch.int32, device=rays.device)
        if ranged:
            self.trace_scene_batch_multi_hits_ranged_into(rays.data_ptr(), m, batch, k, buf.data_ptr(), count.data_ptr())
        else:
            self.trace_scene_batch_multi_hits_into(rays.data_ptr(), m, batch, k, buf.data_ptr(), count.data_ptr(),
                                                   t_min=_or(t_min, 0.0), t_max=_or(t_max, 1e9))
        self.sync()
        return {"t": buf[..., 0], "sphere": buf[..., 1].view(torch.int32), "p": buf[..., 2:5], "normal": buf[..., 5:8],
                "count": count}

    # -- proximity queries (include/ray_b200.h): the spheres within a radius of each ball, nearest first -----------------
    def query_spheres_into(self, balls_dev, n, prepared, k, near_dev, counts_dev=None):
        """The spheres within n balls: balls_dev = device Ball[n] (float[n][4]: centre, r), near_dev = device Near[n][k]
        (d, sphere) in ascending d, then caller index, (+inf, -1) after the last, or None when k == 0; counts_dev =
        device int32[n] (or None) = every sphere within, not capped at k.  Exact against a brute force over every sphere.
        Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_query_spheres(self.handle, prepared.handle, _ptr(balls_dev), int(n), int(k),
                                                    _ptr(near_dev), _ptr(counts_dev)))

    def query_scene_batch_spheres_into(self, balls_dev, m, batch, k, near_dev, counts_dev=None):
        """query_spheres_into for every scene of a SceneBatch: balls_dev = device Ball[B][m], near_dev = device
        Near[B][m][k], counts_dev = device int32[B][m]; sphere indexes the ball's own scene's records.  One launch."""
        self._check(self.lib.ray_b200_scene_batch_query_spheres(self.handle, batch.handle, _ptr(balls_dev), int(m), int(k),
                                                                _ptr(near_dev), _ptr(counts_dev)))

    def query_spheres(self, prepared, balls, k=8):
        """The spheres of a prepared scene within each ball of a [n, 4] float32 CUDA tensor (centre.xyz, r), nearest first:
        dict(d [n, k] float32, sphere [n, k] int32, count [n] int32), views of one [n, k, 2] buffer of Near records and a
        count buffer.  Unused records are d = +inf, sphere = -1; count is not capped at k.  Waits for torch's current
        stream before, and synchronises the context after the query."""
        import torch
        n = proximity_balls(self.device, balls)
        k = proximity_k(k)
        buf = torch.empty((n, k, 2), dtype=torch.float32, device=balls.device)
        count = torch.empty((n,), dtype=torch.int32, device=balls.device)
        torch.cuda.current_stream(balls.device).synchronize()   # the balls may still be in flight on torch's stream
        self.query_spheres_into(balls.data_ptr(), n, prepared, k, buf.data_ptr() if k else None, count.data_ptr())
        self.sync()
        return {"d": buf[..., 0], "sphere": buf[..., 1].view(torch.int32), "count": count}

    def query_scene_batch_spheres(self, batch, balls, k=8):
        """query_spheres for every scene of a SceneBatch: balls is a [B, m, 4] float32 CUDA tensor, m balls per scene.
        Returns dict(d [B, m, k], sphere [B, m, k] int32, count [B, m] int32), sphere indexing the ball's own scene's
        records.  Waits for torch's current stream before, and synchronises the context after the query."""
        import torch
        B = batch.shape[0]
        m = proximity_balls(self.device, balls, B)
        k = proximity_k(k)
        buf = torch.empty((B, m, k, 2), dtype=torch.float32, device=balls.device)
        count = torch.empty((B, m), dtype=torch.int32, device=balls.device)
        torch.cuda.current_stream(balls.device).synchronize()
        self.query_scene_batch_spheres_into(balls.data_ptr(), m, batch, k, buf.data_ptr() if k else None, count.data_ptr())
        self.sync()
        return {"d": buf[..., 0], "sphere": buf[..., 1].view(torch.int32), "count": count}

    # -- nearest-sphere queries (include/ray_b200.h): the k nearest spheres to each point, with or without a limit -------
    def query_nearest_into(self, balls_dev, n, prepared, k, near_dev):
        """The k nearest spheres of n balls: balls_dev = device Ball[n] (float[n][4]: centre, r; r = +inf for no limit),
        near_dev = device Near[n][k] (d, sphere) in ascending d, then caller index, of the spheres with d <= r, (+inf, -1)
        after the last.  Exact against a brute force over every sphere.  Asynchronous on the context's stream."""
        self._check(self.lib.ray_b200_query_nearest(self.handle, prepared.handle, _ptr(balls_dev), int(n), int(k),
                                                    _ptr(near_dev)))

    def query_scene_batch_nearest_into(self, balls_dev, m, batch, k, near_dev):
        """query_nearest_into for every scene of a SceneBatch: balls_dev = device Ball[B][m], near_dev = device
        Near[B][m][k]; sphere indexes the ball's own scene's records.  One launch."""
        self._check(self.lib.ray_b200_scene_batch_query_nearest(self.handle, batch.handle, _ptr(balls_dev), int(m), int(k),
                                                                _ptr(near_dev)))

    def query_nearest(self, prepared, points, k=1):
        """The k nearest spheres of a prepared scene to each point of a [n, 3] float32 CUDA tensor (no limit on the
        distance), or to each ball of a [n, 4] one (centre.xyz, r: only spheres with d <= r): dict(d [n, k] float32,
        sphere [n, k] int32), nearest first, views of one [n, k, 2] buffer of Near records.  Unused records are d = +inf,
        sphere = -1; with no limit a record can have d = +inf (an overflow) and a sphere >= 0.  query_nearest(p, pts)["d"][:, 0]
        is the signed distance of the union of the scene's spheres at each point.  Waits for torch's current stream
        before, and synchronises the context after the query."""
        import torch
        n, balls = nearest_points(self.device, points)
        k = nearest_k(k)
        buf = torch.empty((n, k, 2), dtype=torch.float32, device=balls.device)
        torch.cuda.current_stream(balls.device).synchronize()   # the balls may still be in flight on torch's stream
        self.query_nearest_into(balls.data_ptr(), n, prepared, k, buf.data_ptr())
        self.sync()
        return {"d": buf[..., 0], "sphere": buf[..., 1].view(torch.int32)}

    def query_scene_batch_nearest(self, batch, points, k=1):
        """query_nearest for every scene of a SceneBatch: points is a [B, m, 3] or [B, m, 4] float32 CUDA tensor, m per
        scene.  Returns dict(d [B, m, k], sphere [B, m, k] int32), sphere indexing the point's own scene's records.  Waits
        for torch's current stream before, and synchronises the context after the query."""
        import torch
        B = batch.shape[0]
        m, balls = nearest_points(self.device, points, B)
        k = nearest_k(k)
        buf = torch.empty((B, m, k, 2), dtype=torch.float32, device=balls.device)
        torch.cuda.current_stream(balls.device).synchronize()
        self.query_scene_batch_nearest_into(balls.data_ptr(), m, batch, k, buf.data_ptr())
        self.sync()
        return {"d": buf[..., 0], "sphere": buf[..., 1].view(torch.int32)}

    def count_work(self, h, w, prepared, spp=1):
        wc = WorkCounters()
        self._check(self.lib.ray_b200_count_work(self.handle, int(h), int(w), int(spp), prepared.handle, C.byref(wc)))
        return wc.as_dict()

    def close(self):
        if self.handle:
            self.lib.futhark_context_free(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
