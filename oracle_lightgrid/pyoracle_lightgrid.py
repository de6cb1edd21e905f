"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_lightgrid/liboracle_lightgrid.so: the CPU oracle (oracle/, unchanged) plus the light grid of
ST_OPT_LIGHT_GRID (lightgrid.cpp).  `LightGridOracleEngine` is an `OracleEngine` with `set_light_grid(n)`; with n > 0 it rebuilds the
grid after every tick from the lights its frames see, steps every frame pass by pass and runs the grid version of K5, K13 and K2.
Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_lightgrid.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
P_DI_SAMPLING, P_GI_SAMPLING_B, P_REF_SHADING = 1, 9, 22
K = 64
OVERFLOW = 0xffffffff
HEADER_WORDS = 21
# deliberate mistakes (tests only): of the build (margin, band, the sun) and of K2's pdf
MUTATIONS = {"no_margin": 1, "no_band": 2, "drop_sun": 3, "global_pdf": 4}


def build(force=False):
    srcs = [os.path.join(_DIR, "lightgrid.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "lightgrid.cpp")])
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
        mine.orc_lgrid_create.argtypes, mine.orc_lgrid_create.restype = [], C.c_void_p
        mine.orc_lgrid_destroy.argtypes, mine.orc_lgrid_destroy.restype = [C.c_void_p], None
        mine.orc_lgrid_build.argtypes, mine.orc_lgrid_build.restype = [C.c_void_p, C.c_void_p, C.c_int, C.c_int], None
        mine.orc_lgrid_read.argtypes, mine.orc_lgrid_read.restype = [C.c_void_p, C.c_void_p, C.c_long], C.c_long
        mine.orc_lgrid_point_lists.argtypes = [C.c_void_p, P(np.float32, flags="C"), C.c_long, P(np.uint32, flags="C"), P(np.uint32, flags="C")]
        mine.orc_lgrid_point_lists.restype = None
        mine.orc_lgrid_radiance.argtypes = [C.c_void_p, P(np.float32, flags="C"), P(np.float32, flags="C"), P(np.uint32, flags="C"), C.c_long,
                                            P(np.float32, flags="C")]
        mine.orc_lgrid_radiance.restype = None
        mine.orc_lgrid_step.argtypes, mine.orc_lgrid_step.restype = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int], C.c_int
        _LIB.append(mine)
    return _LIB[0]


def parse(words):
    """st_read_scene("light_grid") / LightGridOracleEngine.read_light_grid() words -> dict of the header, counts and lists."""
    w = np.asarray(words).view(np.uint32)
    f = w[6:HEADER_WORDS].view(np.float32).reshape(5, 3)
    dims = tuple(int(x) for x in w[:3])
    cells = int(w[5])
    counts = w[HEADER_WORDS:HEADER_WORDS + cells + 1]
    lists = w[HEADER_WORDS + cells + 1:].reshape(cells + 1, K)
    return dict(dims=dims, K=int(w[3]), light_count=int(w[4]), cells=cells, lo=f[0], cell=f[1], inv_cell=f[2], band=f[3], margin=f[4],
                counts=counts, lists=lists)


class LightGridOracleEngine(pyoracle.OracleEngine):
    """The oracle with ST_OPT_LIGHT_GRID.  0 (the default) is the oracle.  `mutation` (tests only) applies one deliberate mistake,
    see MUTATIONS."""

    def __init__(self, blue_noise=None, seed_base=0xC0FFEE, mutation=None):
        self.lib = lib()
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}
        self.grid = C.c_void_p(self.lib.orc_lgrid_create())
        self.light_grid = 0
        self._mutation = MUTATIONS[mutation] if mutation else 0

    def __del__(self):
        if getattr(self, "grid", None):
            self.lib.orc_lgrid_destroy(self.grid)
            self.grid = None
        base = getattr(super(), "__del__", None)
        if base:
            base()

    def set_light_grid(self, n):
        """Like st_set_option(ST_OPT_LIGHT_GRID, n): takes effect at the next tick."""
        if not 0 <= int(n) <= 64:
            raise ValueError("light grid: 0 (off) or 1..64")
        self._pending = int(n)

    def tick(self):
        super().tick()
        self.light_grid = getattr(self, "_pending", self.light_grid)
        if self.light_grid:
            self.lib.orc_lgrid_build(self.grid, self.h, self.light_grid, self._mutation)

    def read_light_grid(self):
        n = self.lib.orc_lgrid_read(self.grid, None, 0)
        out = np.empty(n, np.uint32)
        self.lib.orc_lgrid_read(self.grid, out.ctypes.data, n)
        return out

    def point_lists(self, pts):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
        n = np.empty(len(pts), np.uint32)
        ids = np.empty((len(pts), K), np.uint32)
        self.lib.orc_lgrid_point_lists(self.grid, pts, len(pts), n, ids)
        return n, ids

    def radiance(self, pts, nrm, ids):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
        nrm = np.ascontiguousarray(nrm, np.float32).reshape(-1, 3)
        ids = np.ascontiguousarray(ids, np.uint32).reshape(-1)
        out = np.empty((len(pts), 3), np.float32)
        self.lib.orc_lgrid_radiance(self.h, pts, nrm, ids, len(pts), out)
        return out

    def render_camera(self, cam):
        self.render_range(cam, 0, -1)

    def render_range(self, cam, first, last):
        if not self.light_grid:
            return super().render_range(cam, first, last)
        sched = self.frame_schedule(cam)
        last = len(sched) - 1 if last < 0 or last >= len(sched) else last
        for i in range(max(first, 0), last + 1):
            depth = sched[:i].count(P_REF_SHADING)
            if sched[i] in (P_DI_SAMPLING, P_GI_SAMPLING_B) or (sched[i] == P_REF_SHADING and i + 1 < len(sched) and sched[i + 1] != 20):
                assert self.lib.orc_lgrid_step(self.h, self.grid, cam, sched[i], depth, self._mutation) == 0
            else:
                super().render_range(cam, i, i)
