"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_envmap/liboracle_envmap.so: the CPU oracle (oracle/, unchanged) plus the environment map of
st_set_environment_map (envmap.cpp).  `EnvMapOracleEngine` is an `OracleEngine` with `set_environment_map(...)`; while a map is set it
steps every frame pass by pass and runs K10, K13 and K2 with the map in place of the procedural sky, and with
set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1) K12 and K13 draw from the map's distribution.  With no map it is the oracle.
Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_envmap.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
P_DI_RESOLVING, P_GI_SAMPLING_A, P_GI_SAMPLING_B, P_REF_SHADING, P_COMPOSITION = 6, 8, 9, 22, 20
OPT_ENVIRONMENT_MAP_SAMPLING = 19
PROBE_WORDS = 32   # floats per probe record (envmap.cpp documents the layout)
SITE_K10, SITE_K13_MISS, SITE_K13_HIT, SITE_K2 = 0, 1, 2, 3
# deliberate mistakes (tests only): of the lookup, and of K13's sky-draw probability
MUTATIONS = {"v_flip": 1, "phi_zx": 2, "rotation_sign": 3, "clamp_seam": 4, "no_half_texel": 5, "no_intensity": 6, "exposure_x20": 7,
             "sun_gate": 8}
# deliberate mistakes of the sampling (ST_OPT_ENVIRONMENT_MAP_SAMPLING): of the weights, the density, the draw and K12's mixture
SAMPLING_MUTATIONS = {"no_max3": 9, "no_sin_weight": 10, "no_sin_pdf": 11, "draw_rotation_sign": 12, "component_pdf": 13, "no_kappa": 14,
                      "draw_v_flip": 15}


def build(force=False):
    srcs = [os.path.join(_DIR, "envmap.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "envmap.cpp")])
    return LIB


_LIB = []


def lib():
    if not _LIB:
        build()
        mine = C.CDLL(LIB)
        base = pyoracle.lib()
        for name, fn in vars(base).items():   # the oracle's ctypes signatures, for the same functions in this library
            if isinstance(fn, C._CFuncPtr):
                g = getattr(mine, name)
                g.argtypes, g.restype = fn.argtypes, fn.restype
        P = np.ctypeslib.ndpointer
        mine.orc_envm_create.argtypes, mine.orc_envm_create.restype = [], C.c_void_p
        mine.orc_envm_destroy.argtypes, mine.orc_envm_destroy.restype = [C.c_void_p], None
        mine.orc_envm_set.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_float]
        mine.orc_envm_set.restype = C.c_int
        mine.orc_envm_copy.argtypes, mine.orc_envm_copy.restype = [C.c_void_p, C.c_void_p], None
        mine.orc_envm_read.argtypes, mine.orc_envm_read.restype = [C.c_void_p, C.c_void_p, C.c_long], C.c_long
        mine.orc_envm_math.argtypes = [C.c_int, P(np.float32, flags="C"), P(np.float32, flags="C"), P(np.float32, flags="C"), C.c_long]
        mine.orc_envm_math.restype = None
        mine.orc_envm_sample.argtypes = [C.c_void_p, P(np.float32, flags="C"), C.c_long, C.c_int, P(np.float32, flags="C")]
        mine.orc_envm_sample.restype = None
        mine.orc_envm_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long]
        mine.orc_envm_apply.restype = C.c_long
        mine.orc_envm_distribution.argtypes, mine.orc_envm_distribution.restype = [C.c_void_p, C.c_int, C.c_int], C.c_float
        mine.orc_envm_read_distribution.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
        mine.orc_envm_read_distribution.restype = C.c_long
        mine.orc_envm_draw.argtypes = [C.c_void_p, P(np.float32, flags="C"), C.c_long, C.c_int, P(np.float32, flags="C"), P(np.uint32, flags="C")]
        mine.orc_envm_draw.restype = None
        mine.orc_envm_pdf.argtypes = [C.c_void_p, P(np.float32, flags="C"), C.c_long, C.c_int, P(np.float32, flags="C")]
        mine.orc_envm_pdf.restype = None
        mine.orc_envm_surface_draws.argtypes = [C.c_void_p, C.c_int, P(np.float32, flags="C"), P(np.uint32, flags="C"), C.c_long, C.c_int,
                                                P(np.float32, flags="C")]
        mine.orc_envm_surface_draws.restype = None
        _LIB.append(mine)
    return _LIB[0]


def envm_math(op, a, b=None):
    """st_device_math ops 8 (acos) and 9 (atan2(a, b)) as the oracle evaluates them."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1)
    b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, np.float32).reshape(-1)
    out = np.empty_like(a)
    lib().orc_envm_math(op, a, b, out, a.size)
    return out


def parse(words):
    """st_read_scene("environment_map") / EnvMapOracleEngine.read_environment_map() words -> (W, H, intensity, rotation, texels [H, W, 4])."""
    w = np.asarray(words, np.float32)
    u = w.view(np.uint32)
    W, H = int(u[0]), int(u[1])
    return W, H, float(w[2]), float(w[3]), w[4:4 + 4 * W * H].reshape(H, W, 4)


def parse_distribution(words):
    """st_read_scene("environment_map_distribution") words -> (W, H, total, marginal CDF [H], conditional CDFs [H, W])."""
    w = np.asarray(words, np.float32)
    W, H = int(w[:2].view(np.uint32)[0]), int(w[:2].view(np.uint32)[1])
    return W, H, w[2], w[3:3 + H], w[3 + H:3 + H + W * H].reshape(H, W)


class EnvMap:
    """A map and its distribution on their own (no engine): the lookup, env_draw, env_pdf and the K12 / K13 draws at one surface, in
    the oracle's arithmetic.  `mutation` (tests only): one of MUTATIONS or SAMPLING_MUTATIONS."""

    def __init__(self, rgba, intensity=1.0, rotation=0.0, mutation=None):
        self.lib = lib()
        self.m = C.c_void_p(self.lib.orc_envm_create())
        t = _texels(rgba)
        if self.lib.orc_envm_set(self.m, t.ctypes.data, t.shape[1], t.shape[0], intensity, rotation) != 0:
            raise ValueError("invalid environment map")
        self.mut = {**MUTATIONS, **SAMPLING_MUTATIONS}[mutation] if mutation else 0
        self.total = self.lib.orc_envm_distribution(self.m, 1, self.mut)

    def __del__(self):
        if getattr(self, "m", None):
            self.lib.orc_envm_destroy(self.m)
            self.m = None

    def distribution(self):
        n = self.lib.orc_envm_read_distribution(self.m, None, 0)
        out = np.empty(n, np.float32)
        self.lib.orc_envm_read_distribution(self.m, out.ctypes.data, n)
        return parse_distribution(out)

    def draw(self, xi):
        """env_draw for n x 2 (xi1, xi2) -> (n x 3 directions, n x 2 (row, column) cells)."""
        xi = np.ascontiguousarray(xi, np.float32).reshape(-1, 2)
        out = np.empty((xi.shape[0], 3), np.float32)
        cells = np.empty((xi.shape[0], 2), np.uint32)
        self.lib.orc_envm_draw(self.m, xi.reshape(-1), xi.shape[0], self.mut, out.reshape(-1), cells.reshape(-1))
        return out, cells

    def pdf(self, dirs):
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        out = np.empty(d.shape[0], np.float32)
        self.lib.orc_envm_pdf(self.m, d.reshape(-1), d.shape[0], self.mut, out)
        return out

    def sample(self, dirs):
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        out = np.empty_like(d)
        self.lib.orc_envm_sample(self.m, d.reshape(-1), d.shape[0], 0, out.reshape(-1))
        return out

    def surface_draws(self, k13, normal, view, metallic, roughness, seeds):
        """K12's mixture draw (k13 False) or K13's sky draw (k13 True) at one surface, one WhiteNoise per seed: n x 8 records
        {direction, K12: q / kappa | K13: 1 where below the surface, K12: the map's value | K13: the sky-draw value, 0}."""
        nvmr = np.array(list(normal) + list(view) + [metallic, roughness], np.float32)
        seeds = np.ascontiguousarray(seeds, np.uint32)
        out = np.empty((seeds.size, 8), np.float32)
        self.lib.orc_envm_surface_draws(self.m, int(k13), nvmr, seeds, seeds.size, self.mut, out.reshape(-1))
        return out


def _texels(rgba):
    a = np.asarray(rgba, dtype=np.float32)
    if a.shape[2] == 3:
        a = np.concatenate([a, np.ones(a.shape[:2] + (1,), np.float32)], axis=2)
    return np.ascontiguousarray(a)


class EnvMapOracleEngine(pyoracle.OracleEngine):
    """The oracle with st_set_environment_map.  With no map (the default) it is the oracle.  `mutation` (tests only) applies one
    deliberate mistake, see MUTATIONS."""

    def __init__(self, blue_noise=None, seed_base=0xC0FFEE, mutation=None):
        self.lib = lib()
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}
        self.pending = C.c_void_p(self.lib.orc_envm_create())   # the map as last set
        self.em = C.c_void_p(self.lib.orc_envm_create())        # the map as the last tick took it
        self.map_on = False
        self._pending_on = False
        self._mutation = {**MUTATIONS, **SAMPLING_MUTATIONS}[mutation] if mutation else 0
        self.probes = None   # a list to collect (pass, depth, records) into, or None
        self.sampling = False        # OPT_ENVIRONMENT_MAP_SAMPLING as set
        self.sampled = False         # the last tick's frames draw from the map's distribution

    def __del__(self):
        for k in ("pending", "em"):
            if getattr(self, k, None):
                self.lib.orc_envm_destroy(getattr(self, k))
                setattr(self, k, None)
        base = getattr(super(), "__del__", None)
        if base:
            base()

    def set_environment_map(self, rgba=None, intensity=1.0, rotation=0.0):
        """Like st_set_environment_map: validated now (ValueError, nothing changes), taken at the next tick."""
        if rgba is None:
            self.lib.orc_envm_set(self.pending, None, 0, 0, 0.0, 0.0)
            self._pending_on = False
            return
        t = _texels(rgba)
        if self.lib.orc_envm_set(self.pending, t.ctypes.data, t.shape[1], t.shape[0], intensity, rotation) != 0:
            raise ValueError("invalid environment map")
        self._pending_on = True

    def set_option(self, option, value):
        """OPT_ENVIRONMENT_MAP_SAMPLING (0 or 1, else ValueError), taken at the next tick; the oracle has no other option."""
        if option != OPT_ENVIRONMENT_MAP_SAMPLING or value not in (0, 1):
            raise ValueError(f"option {option} = {value}")
        self.sampling = bool(value)

    def tick(self):
        super().tick()
        self.map_on = self._pending_on
        self.lib.orc_envm_copy(self.em, self.pending)
        total = self.lib.orc_envm_distribution(self.em, int(self.sampling and self.map_on), self._mutation)
        self.sampled = self.sampling and self.map_on and 0.0 < total < float("inf")

    def read_distribution(self):
        n = self.lib.orc_envm_read_distribution(self.em, None, 0)
        out = np.empty(n, np.float32)
        if n:
            self.lib.orc_envm_read_distribution(self.em, out.ctypes.data, n)
        return out

    def read_environment_map(self):
        n = self.lib.orc_envm_read(self.em, None, 0) if self.map_on else 0
        out = np.empty(n, np.float32)
        if n:
            self.lib.orc_envm_read(self.em, out.ctypes.data, n)
        return out

    def sample(self, dirs, mutation=None):
        """The lookup of the map the last tick took, for n directions (n x 3) -> n x 3 radiances."""
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        out = np.empty_like(d)
        self.lib.orc_envm_sample(self.em, d.reshape(-1), d.shape[0], MUTATIONS[mutation] if mutation else self._mutation, out.reshape(-1))
        return out

    def render_camera(self, cam):
        self.render_range(cam, 0, -1)

    def render_range(self, cam, first, last):
        if not self.map_on:
            return super().render_range(cam, first, last)
        sched = self.frame_schedule(cam)
        last = len(sched) - 1 if last < 0 or last >= len(sched) else last
        for i in range(max(first, 0), last + 1):
            p = sched[i]
            ref_step = p == P_REF_SHADING and i + 1 < len(sched) and sched[i + 1] != P_COMPOSITION
            if p in (P_DI_RESOLVING, P_GI_SAMPLING_B) or ref_step or (p == P_GI_SAMPLING_A and self.sampled):
                depth = sched[:i].count(P_REF_SHADING) if ref_step else 0
                self._apply(cam, p, depth)
                continue
            super().render_range(cam, i, i)

    def _apply(self, cam, pass_id, depth):
        if self.probes is None:
            assert self.lib.orc_envm_apply(self.h, self.em, cam, pass_id, depth, self._mutation, None, 0) >= 0
            return
        n = self.read_buffer(cam, "output").size // 4   # one record per pixel at most
        out = np.empty(n * PROBE_WORDS, np.float32)
        k = self.lib.orc_envm_apply(self.h, self.em, cam, pass_id, depth, self._mutation, out.ctypes.data, out.size)
        assert k >= 0, k
        self.probes.append((pass_id, depth, out[:k * PROBE_WORDS].reshape(k, PROBE_WORDS).copy()))
