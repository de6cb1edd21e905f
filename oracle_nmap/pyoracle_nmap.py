"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_nmap/liboracle_nmap.so: the CPU oracle (oracle/, unchanged) plus the normal-mapping rule of
ST_OPT_NORMAL_MAPS applied at K0, K12 and K1 (nmap.cpp).  `NormalMapOracleEngine` is an `OracleEngine` with
`set_normal_maps(on)`; with the option on it steps every frame pass by pass and applies the rule after those three passes.
Imported only by tests/.
"""
import ctypes as C
import os
import subprocess

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_nmap.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
P_PRIM_GBUFFER, P_GI_SAMPLING_A, P_REF_TRACING = 0, 8, 21
MUTATIONS = {"srgb_decode": 1, "cross_order": 2, "no_backface_sign": 3, "renormalise_tangent": 4, "no_fallback": 5}


def build(force=False):
    srcs = [os.path.join(_DIR, "nmap.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "nmap.cpp")])
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
        mine.orc_nmap_apply.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        mine.orc_nmap_apply.restype = C.c_int
        _LIB.append(mine)
    return _LIB[0]


class NormalMapOracleEngine(pyoracle.OracleEngine):
    """The oracle with ST_OPT_NORMAL_MAPS.  Off (the default) it is the oracle.  `mutation` (tests only) applies one deliberate
    mistake to the rule, see MUTATIONS."""

    def __init__(self, blue_noise=None, seed_base=0xC0FFEE, mutation=None):
        self.lib = lib()
        import numpy as np
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}
        self.normal_maps = False
        self._mutation = MUTATIONS[mutation] if mutation else 0

    def set_normal_maps(self, on):
        self.normal_maps = bool(on)

    def render_camera(self, cam):
        self.render_range(cam, 0, -1)

    def render_range(self, cam, first, last):
        if not self.normal_maps:
            return super().render_range(cam, first, last)
        sched = self.frame_schedule(cam)
        last = len(sched) - 1 if last < 0 or last >= len(sched) else last
        for i in range(max(first, 0), last + 1):
            super().render_range(cam, i, i)
            if sched[i] in (P_PRIM_GBUFFER, P_GI_SAMPLING_A, P_REF_TRACING):
                depth = sched[:i].count(P_REF_TRACING)
                assert self.lib.orc_nmap_apply(self.h, cam, sched[i], depth, self._mutation) == 0
