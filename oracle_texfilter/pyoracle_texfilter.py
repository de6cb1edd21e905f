"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_texfilter/liboracle_texfilter.so: the CPU oracle (oracle/, unchanged) plus the texture filter of
ST_OPT_TEXTURE_FILTER (texfilter.cpp).  `TextureFilterOracleEngine` is an `OracleEngine` with `set_texture_filter(on)`; with the option
on it rebuilds the mip chains after every tick, steps every frame pass by pass, patches the material terms K0 and K12 stored, and runs
the filtered K2.  Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_texfilter.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
P_PRIM_GBUFFER, P_GI_SAMPLING_A, P_REF_SHADING, P_COMPOSITION = 0, 8, 22, 20
PROBE_WORDS = 40   # floats per orc_texf_probe record
# deliberate mistakes (tests only): of the mip build, of the level of detail, of the taps and of the level blend
MUTATIONS = {"raw_bytes": 1, "no_cos": 2, "clamp_atlas": 3, "no_half_texel": 4, "swap_levels": 5}


def build(force=False):
    srcs = [os.path.join(_DIR, "texfilter.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "texfilter.cpp")])
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
        mine.orc_texf_create.argtypes, mine.orc_texf_create.restype = [], C.c_void_p
        mine.orc_texf_destroy.argtypes, mine.orc_texf_destroy.restype = [C.c_void_p], None
        mine.orc_texf_build.argtypes, mine.orc_texf_build.restype = [C.c_void_p, C.c_void_p, C.c_int], None
        mine.orc_texf_remove_image.argtypes, mine.orc_texf_remove_image.restype = [C.c_void_p, C.c_uint64], None
        mine.orc_texf_read.argtypes, mine.orc_texf_read.restype = [C.c_void_p, C.c_void_p, C.c_long], C.c_long
        mine.orc_texf_srgb_lut.argtypes, mine.orc_texf_srgb_lut.restype = [C.c_void_p, P(np.float32, flags="C")], None
        mine.orc_texf_log2.argtypes, mine.orc_texf_log2.restype = [P(np.float32, flags="C"), P(np.float32, flags="C"), C.c_long], None
        mine.orc_texf_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long]
        mine.orc_texf_probe.restype = C.c_long
        mine.orc_texf_apply.argtypes, mine.orc_texf_apply.restype = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int], C.c_int
        _LIB.append(mine)
    return _LIB[0]


def log2_lod(a):
    """The level of detail's log2 as the oracle evaluates it (st_device_math op 7 on the device)."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1)
    out = np.empty_like(a)
    lib().orc_texf_log2(a, out, a.size)
    return out


def parse(words):
    """st_read_scene("texture_mips") / TextureFilterOracleEngine.read_texture_mips() words -> (table [materials, 3, 2], pool [T, 4] bytes)."""
    w = np.asarray(words).view(np.uint32)
    texels, mats = int(w[0]), int(w[1])
    table = w[2:2 + 6 * mats].reshape(mats, 3, 2)
    pool = w[2 + 6 * mats:2 + 6 * mats + texels].copy().view(np.uint8).reshape(texels, 4)
    return table, pool


class TextureFilterOracleEngine(pyoracle.OracleEngine):
    """The oracle with ST_OPT_TEXTURE_FILTER.  Off (the default) it is the oracle.  `mutation` (tests only) applies one deliberate
    mistake, see MUTATIONS."""

    def __init__(self, blue_noise=None, seed_base=0xC0FFEE, mutation=None):
        self.lib = lib()
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}
        self.tf = C.c_void_p(self.lib.orc_texf_create())
        self.texture_filter = False
        self._mutation = MUTATIONS[mutation] if mutation else 0

    def __del__(self):
        if getattr(self, "tf", None):
            self.lib.orc_texf_destroy(self.tf)
            self.tf = None
        base = getattr(super(), "__del__", None)
        if base:
            base()

    def set_texture_filter(self, on):
        """Like st_set_option(ST_OPT_TEXTURE_FILTER, on): takes effect at the next tick."""
        self._pending = bool(on)

    def remove_image(self, handle):
        self.lib.orc_texf_remove_image(self.h, handle)

    def tick(self):
        super().tick()
        self.texture_filter = getattr(self, "_pending", self.texture_filter)
        if self.texture_filter:
            self.lib.orc_texf_build(self.tf, self.h, self._mutation)

    def srgb_lut(self):
        """The 256-entry sRGB -> linear table (after the first insert_image)."""
        out = np.zeros(256, np.float32)
        self.lib.orc_texf_srgb_lut(self.h, out)
        return out

    def read_texture_mips(self):
        n = self.lib.orc_texf_read(self.tf, None, 0)
        out = np.empty(n, np.uint32)
        self.lib.orc_texf_read(self.tf, out.ctypes.data, n)
        return out

    def probe(self, cam, pass_id, depth=0):
        """orc_texf_probe's records (n, PROBE_WORDS) for step `pass_id` of the current frame (texfilter.cpp documents the layout)."""
        n = self.lib.orc_texf_probe(self.h, self.tf, cam, pass_id, depth, self._mutation, None, 0)
        assert n >= 0, n
        out = np.empty((n, PROBE_WORDS), np.float32)
        assert self.lib.orc_texf_probe(self.h, self.tf, cam, pass_id, depth, self._mutation, out.ctypes.data, out.size) == n
        return out

    def render_camera(self, cam):
        self.render_range(cam, 0, -1)

    def render_range(self, cam, first, last):
        if not self.texture_filter:
            return super().render_range(cam, first, last)
        sched = self.frame_schedule(cam)
        last = len(sched) - 1 if last < 0 or last >= len(sched) else last
        for i in range(max(first, 0), last + 1):
            depth = sched[:i].count(P_REF_SHADING)
            if sched[i] == P_REF_SHADING and i + 1 < len(sched) and sched[i + 1] != P_COMPOSITION:
                assert self.lib.orc_texf_apply(self.h, self.tf, cam, P_REF_SHADING, depth, self._mutation) == 0
                continue
            super().render_range(cam, i, i)
            if sched[i] in (P_PRIM_GBUFFER, P_GI_SAMPLING_A):
                assert self.lib.orc_texf_apply(self.h, self.tf, cam, sched[i], 0, self._mutation) == 0
