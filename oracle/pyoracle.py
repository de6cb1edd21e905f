"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle/liboracle.so (CPU restatement of the reference hot
path).  Imported only by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))


def build(force=False):
    """Compile the oracle (g++, seconds).  Building the checker is not using it."""
    libs = [os.path.join(_DIR, n) for n in ("liboracle.so", "liboracle_libm.so")]
    srcs = [os.path.join(_DIR, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp", "Makefile")]
    newest = max(os.path.getmtime(s) for s in srcs)
    if force or any((not os.path.exists(l)) or os.path.getmtime(l) < newest for l in libs):
        subprocess.check_call(["make", "-C", _DIR, "-j2"], stdout=subprocess.DEVNULL)
    return libs


_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")


def _load(libm=False):
    build()
    lib = C.CDLL(os.path.join(_DIR, "liboracle_libm.so" if libm else "liboracle.so"))
    lib.orc_engine_create.restype = C.c_void_p
    sig = {
        "orc_engine_destroy": [C.c_void_p],
        "orc_set_blue_noise": [C.c_void_p, _u8p],
        "orc_set_seed_base": [C.c_void_p, C.c_uint32],
        "orc_insert_mesh": [C.c_void_p, C.c_uint64, _f32p, C.c_int],
        "orc_insert_material": [C.c_void_p, C.c_uint64, _f32p, C.c_int],
        "orc_insert_image": [C.c_void_p, C.c_uint64, _u8p, C.c_int, C.c_int],
        "orc_set_material_textures": [C.c_void_p, C.c_uint64, np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS"), C.c_uint32],
        "orc_insert_instance": [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, _f32p],
        "orc_remove_instance": [C.c_void_p, C.c_uint64],
        "orc_insert_light": [C.c_void_p, C.c_uint64, C.c_int, _f32p],
        "orc_remove_light": [C.c_void_p, C.c_uint64],
        "orc_update_sun": [C.c_void_p, C.c_float, C.c_float],
        "orc_create_camera": [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, _f32p],
        "orc_update_camera": [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, _f32p],
        "orc_tick": [C.c_void_p],
        "orc_render_camera": [C.c_void_p, C.c_int],
        "orc_render_range": [C.c_void_p, C.c_int, C.c_int, C.c_int],
        "orc_frame_schedule": [C.c_void_p, C.c_int, C.c_void_p, C.c_int],
        "orc_read_buffer": [C.c_void_p, C.c_int, C.c_char_p, C.c_void_p, C.c_long],
        "orc_read_scene": [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long],
        "orc_bvh_depth": [C.c_void_p],
        "orc_trace_closest": [C.c_void_p, _f32p, C.c_long, _f32p],
        "orc_trace_any": [C.c_void_p, _f32p, C.c_long, _u32p],
        "orc_trace_brute": [C.c_void_p, _f32p, C.c_long, _f32p, _u32p],
        "orc_math": [C.c_int, _f32p, _f32p, _f32p, C.c_long],
        "orc_gbuffer_pack": [_f32p, _f32p],
        "orc_gbuffer_unpack": [_f32p, _f32p],
        "orc_camera_contain": [C.c_float, C.c_float, C.c_int, C.c_int, _u32p],
        "orc_di_reservoir_roundtrip": [_f32p, C.c_long, _f32p, _f32p],
        "orc_reprojection_roundtrip": [_f32p, C.c_uint32, _f32p, _u32p],
        "orc_allocator_script": [_i64p, C.c_int, _i64p],
        "orc_bvh_builder_destroy": [C.c_void_p],
        "orc_bvh_builder_build": [C.c_void_p, _f32p, C.c_long, C.c_int, C.c_void_p, C.c_long, C.POINTER(C.c_uint32), C.POINTER(C.c_int)],
        "orc_set_bvh_reuse": [C.c_void_p, C.c_int],
    }
    for name, args in sig.items():
        getattr(lib, name).argtypes = args
    lib.orc_read_buffer.restype = C.c_long
    lib.orc_bvh_builder_create.restype = C.c_void_p
    lib.orc_bvh_builder_build.restype = C.c_long
    lib.orc_bvh_reused.restype = C.c_uint32
    lib.orc_bvh_reused.argtypes = [C.c_void_p]
    lib.orc_read_scene.restype = C.c_long
    lib.orc_u32_bytes_roundtrip.restype = C.c_uint32
    lib.orc_u32_bytes_roundtrip.argtypes = [C.c_uint32]
    lib.orc_ray_count.restype = C.c_uint64
    lib.orc_ray_count.argtypes = [C.c_int]
    lib.orc_set_threads.argtypes = [C.c_int]
    lib.orc_get_threads.restype = C.c_int
    lib.orc_frame.restype = C.c_uint32
    lib.orc_frame.argtypes = [C.c_void_p]
    return lib


_LIBS = {}


def lib(libm=False):
    if libm not in _LIBS:
        _LIBS[libm] = _load(libm)
    return _LIBS[libm]


def _f(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1))


class OracleBvhBuilder:
    """strolle/src/bvh/builder.rs + serializer.rs on their own; same interface as strolle_b200.engine.BvhBuilder."""

    def __init__(self, libm=False):
        self.lib = lib(libm)
        self._h = C.c_void_p(self.lib.orc_bvh_builder_create())
        self.grafted = 0
        self.depth = 0

    def build(self, prims, reuse=True):
        prims = np.ascontiguousarray(prims, dtype=np.float32).reshape(-1, 11)
        g = C.c_uint32(0); d = C.c_int(0)
        cap = max(16, prims.shape[0] * 4 * 4 * 2 + 16)   # <= n leaf entries + (n - 1) internal nodes of 4 float4 each
        out = np.zeros(cap, dtype=np.float32)
        n = self.lib.orc_bvh_builder_build(self._h, prims.reshape(-1), prims.shape[0], int(reuse), out.ctypes.data, cap, C.byref(g), C.byref(d))
        assert n <= cap
        self.grafted, self.depth = int(g.value), int(d.value)
        return out[:n].reshape(-1, 4).copy()

    def __del__(self):
        try:
            self.lib.orc_bvh_builder_destroy(self._h)
        except Exception:
            pass


class OracleEngine:
    """Mirror of strolle::Engine (strolle/src/lib.rs:104-395) over the CPU oracle."""

    def __init__(self, libm=False, blue_noise=None, seed_base=0xC0FFEE):
        self.lib = lib(libm)
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}

    def close(self):
        if self.h:
            self.lib.orc_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def insert_mesh(self, handle, triangles36):
        t = _f(triangles36)
        self.lib.orc_insert_mesh(self.h, handle, t, t.size // 36)

    def insert_material(self, handle, params12, alpha_blend=False):
        self.lib.orc_insert_material(self.h, handle, _f(params12), int(alpha_blend))

    def insert_image(self, handle, rgba8):
        a = np.ascontiguousarray(rgba8, dtype=np.uint8)
        h, w = a.shape[0], a.shape[1]
        if self.lib.orc_insert_image(self.h, handle, a.reshape(-1), w, h) != 0:
            raise RuntimeError("atlas full")

    def set_material_textures(self, handle, base_color=None, emissive=None, metallic_roughness=None, normal_map=None):
        t = [base_color, emissive, metallic_roughness, normal_map]
        mask = sum((1 << i) for i, v in enumerate(t) if v is not None)
        self.lib.orc_set_material_textures(self.h, handle, np.array([v or 0 for v in t], dtype=np.uint64), mask)

    def insert_instance(self, handle, mesh, material, affine12):
        self.lib.orc_insert_instance(self.h, handle, mesh, material, _f(affine12))

    def remove_instance(self, handle):
        self.lib.orc_remove_instance(self.h, handle)

    def insert_light(self, handle, kind, params12):
        self.lib.orc_insert_light(self.h, handle, kind, _f(params12))

    def remove_light(self, handle):
        self.lib.orc_remove_light(self.h, handle)

    def update_sun(self, azimuth, altitude):
        self.lib.orc_update_sun(self.h, azimuth, altitude)

    def create_camera(self, mode, denoise, ref_depth, w, h, transform16, projection16):
        cam = self.lib.orc_create_camera(self.h, mode, int(denoise), ref_depth, w, h, _f(transform16), _f(projection16))
        self._cams[cam] = (w, h)
        return cam

    def update_camera(self, cam, mode, denoise, ref_depth, w, h, transform16, projection16):
        self.lib.orc_update_camera(self.h, cam, mode, int(denoise), ref_depth, w, h, _f(transform16), _f(projection16))
        self._cams[cam] = (w, h)

    def tick(self):
        self.lib.orc_tick(self.h)

    def render_camera(self, cam):
        self.lib.orc_render_camera(self.h, cam)

    def render_range(self, cam, first, last):
        """Steps [first, last] of this frame's schedule (last < 0: to the end); same step list as the CUDA engine's strict,
        unfused schedule."""
        self.lib.orc_render_range(self.h, cam, first, last)

    def frame_schedule(self, cam):
        """Pass ids (the CUDA engine's PassId values) of this frame's steps."""
        ids = (C.c_int * 64)()
        n = self.lib.orc_frame_schedule(self.h, cam, ids, 64)
        return list(ids[:n])

    def read_buffer(self, cam, name):
        n = self.lib.orc_read_buffer(self.h, cam, name.encode(), None, 0)
        if n < 0:
            raise KeyError(name)
        out = np.empty(n, dtype=np.float32)
        self.lib.orc_read_buffer(self.h, cam, name.encode(), out.ctypes.data_as(C.c_void_p), n)
        return out

    def read_scene(self, name):
        n = self.lib.orc_read_scene(self.h, name.encode(), None, 0)
        if n < 0:
            raise KeyError(name)
        out = np.empty(n, dtype=np.float32)
        self.lib.orc_read_scene(self.h, name.encode(), out.ctypes.data_as(C.c_void_p), n)
        return out

    def set_bvh_reuse(self, reuse):
        self.lib.orc_set_bvh_reuse(self.h, int(reuse))

    def bvh_reused(self):
        return int(self.lib.orc_bvh_reused(self.h))

    def bvh_depth(self):
        return self.lib.orc_bvh_depth(self.h)

    def trace_closest(self, rays8):
        r = _f(rays8)
        n = r.size // 8
        out = np.empty(n * 12, dtype=np.float32)
        self.lib.orc_trace_closest(self.h, r, n, out)
        return out.reshape(n, 12)

    def trace_any(self, rays8):
        r = _f(rays8)
        n = r.size // 8
        out = np.empty(n, dtype=np.uint32)
        self.lib.orc_trace_any(self.h, r, n, out)
        return out

    def trace_brute(self, rays8):
        r = _f(rays8)
        n = r.size // 8
        d = np.empty(n, dtype=np.float32)
        t = np.empty(n, dtype=np.uint32)
        self.lib.orc_trace_brute(self.h, r, n, d, t)
        return d, t


def usable_cpus():
    """CPUs this process may actually use: affinity mask capped by the cgroup CPU quota."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = max(1, min(n, int(float(quota) / float(period) + 0.5)))
    except Exception:
        pass
    return n


def set_threads(n=None, libm=False):
    """Sets the oracle's OpenMP thread count (default: usable_cpus()); returns the count in effect."""
    l = lib(libm)
    l.orc_set_threads(int(n if n else usable_cpus()))
    return int(l.orc_get_threads())


def ray_count(reset=False, libm=False):
    return int(lib(libm).orc_ray_count(int(reset)))


def math(op, a, b=None, libm=False):
    ops = {"sin": 0, "cos": 1, "acos": 2, "atan2": 3, "exp": 4, "pow": 5, "acos_approx": 6, "f16": 7}
    a = _f(a)
    b = _f(b) if b is not None else np.zeros_like(a)
    out = np.empty_like(a)
    lib(libm).orc_math(ops[op], a, b, out, a.size)
    return out
