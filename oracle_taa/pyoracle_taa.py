"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_taa/liboracle_taa.so: the CPU oracle (oracle/, unchanged) plus the camera jitter and the temporal resolve
of ST_OPT_TEMPORAL_AA (taa.cpp).  `TemporalAAOracleEngine` is an `OracleEngine` with `set_temporal_aa(on)`; with the option on it renders
every frame through the jittered cameras and resolves the composed frame against the camera's history, as the device does.  Imported
only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_taa.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
P_COMPOSITION = 20
MODE_BVH_HEATMAP, MODE_REFERENCE = 5, 6
PROBE_WORDS = 24   # floats per pixel of orc_taa_resolve's probe (taa.cpp documents the layout)
# deliberate mistakes (tests only): of the history position, the jitter, the clip, the tonemap, the blend, the filter, the sky
MUTATIONS = {"no_jitter_diff": 1, "y_sign": 2, "clamp": 3, "no_tonemap": 4, "fixed_alpha": 5, "bilinear": 6, "sky_point": 7}


def build(force=False):
    srcs = [os.path.join(_DIR, "taa.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "taa.cpp")])
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
        F = np.ctypeslib.ndpointer(np.float32, flags="C")
        mine.orc_taa_jitter.argtypes, mine.orc_taa_jitter.restype = [C.c_uint, F], None
        mine.orc_taa_set_cameras.argtypes, mine.orc_taa_set_cameras.restype = [C.c_void_p, C.c_int, F, F, C.c_int, C.c_int], C.c_int
        mine.orc_taa_resolve.argtypes, mine.orc_taa_resolve.restype = [C.c_void_p, C.c_int, F, F, C.c_int, C.c_void_p], C.c_int
        mine.orc_taa_resolve_arrays.argtypes = [C.c_int] * 4 + [F] * 12 + [F, F]
        mine.orc_taa_resolve_arrays.restype = C.c_int
        _LIB.append(mine)
    return _LIB[0]


def jitter(frame):
    """J(frame) in pixels, as float32 (x, y)."""
    out = np.zeros(2, np.float32)
    lib().orc_taa_jitter(frame & 0xffffffff, out)
    return out


def resolve_arrays(w, h, mode, cur, bufs, cam_curr, cam_prev, jit4, hist_in):
    """The resolve over a device's own inputs.  bufs: d0, d1 (the current G-buffer), di_diff, di_spec, gi_diff, gi_spec (the final
    signals the composition reads), ref_colors, vel, each (w * h * 4) float32.  Returns (history, output)."""
    f = lambda a: np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1))
    hist_out, out = np.zeros(w * h * 4, np.float32), np.zeros(w * h * 4, np.float32)
    names = ("d0", "d1", "di_diff", "di_spec", "gi_diff", "gi_spec", "ref_colors", "vel")
    assert lib().orc_taa_resolve_arrays(w, h, mode, cur, *[f(bufs[k]) for k in names], f(cam_curr), f(cam_prev), f(jit4), f(hist_in), hist_out, out) == 0
    return hist_out, out


class TemporalAAOracleEngine(pyoracle.OracleEngine):
    """The oracle with ST_OPT_TEMPORAL_AA.  Off (the default) it is the oracle.  `mutation` (tests only) applies one deliberate
    mistake, see MUTATIONS."""

    def __init__(self, blue_noise=None, seed_base=0xC0FFEE, mutation=None):
        self.lib = lib()
        self.h = C.c_void_p(self.lib.orc_engine_create())
        if blue_noise is not None:
            self.lib.orc_set_blue_noise(self.h, np.ascontiguousarray(blue_noise, dtype=np.uint8).reshape(-1))
        self.lib.orc_set_seed_base(self.h, seed_base)
        self._cams = {}
        self._desc, self._prev, self._jittered, self._hist = {}, {}, set(), {}
        self.temporal_aa = False
        self._mutation = MUTATIONS[mutation] if mutation else 0
        self.probe = None   # set to True to keep the last resolve's per-pixel record (PROBE_WORDS floats) in self.last_probe

    def set_temporal_aa(self, on):
        """Like st_set_option(ST_OPT_TEMPORAL_AA, on): takes effect at the next tick."""
        self._pending = bool(on)

    def create_camera(self, mode, denoise, ref_depth, w, h, transform16, projection16):
        cam = super().create_camera(mode, denoise, ref_depth, w, h, transform16, projection16)
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h, pyoracle._f(transform16), pyoracle._f(projection16))
        self._prev[cam] = self._desc[cam]
        return cam

    def update_camera(self, cam, mode, denoise, ref_depth, w, h, transform16, projection16):
        self._unjitter(cam)   # the oracle's prev = curr must see the unjittered camera
        old = self._desc[cam]
        self._prev[cam] = old
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h, pyoracle._f(transform16), pyoracle._f(projection16))
        if old[:5] != self._desc[cam][:5]:
            self._hist.pop(cam, None)   # camera reallocation: the history starts over
        super().update_camera(cam, mode, denoise, ref_depth, w, h, transform16, projection16)

    def _unjitter(self, cam):
        if cam in self._jittered:
            p = self._prev[cam]
            self.lib.orc_taa_set_cameras(self.h, cam, p[5], p[6], 0, 0)
            self._jittered.discard(cam)

    def tick(self):
        for cam in list(self._jittered):
            self._unjitter(cam)
        super().tick()
        on = getattr(self, "_pending", self.temporal_aa)
        if on != self.temporal_aa:
            self._hist.clear()   # freed when the option turns off, zero when it turns on
        self.temporal_aa = on

    def _active(self, cam):
        return self.temporal_aa and self._desc[cam][0] not in (MODE_BVH_HEATMAP, MODE_REFERENCE)

    def history(self, cam):
        """(taa_history_a, taa_history_b) as float32 arrays."""
        if cam not in self._hist:
            w, h = self._desc[cam][3], self._desc[cam][4]
            self._hist[cam] = (np.zeros(w * h * 4, np.float32), np.zeros(w * h * 4, np.float32))
        return self._hist[cam]

    def read_buffer(self, cam, name):
        if name in ("taa_history_a", "taa_history_b"):
            if cam not in self._hist:
                raise KeyError(name)
            return self._hist[cam][0 if name.endswith("a") else 1].copy()
        return super().read_buffer(cam, name)

    def render_camera(self, cam):
        self.render_range(cam, 0, -1)

    def render_range(self, cam, first, last):
        if not self._active(cam):
            return super().render_range(cam, first, last)
        p = self._prev[cam]
        self.lib.orc_taa_set_cameras(self.h, cam, p[5], p[6], 1, self._mutation)
        self._jittered.add(cam)
        sched = self.frame_schedule(cam)
        last = len(sched) - 1 if last < 0 or last >= len(sched) else last
        for i in range(max(first, 0), last + 1):
            super().render_range(cam, i, i)
            if sched[i] == P_COMPOSITION:
                ha, hb = self.history(cam)
                probe = np.zeros(self._desc[cam][3] * self._desc[cam][4] * PROBE_WORDS, np.float32) if self.probe else None
                assert self.lib.orc_taa_resolve(self.h, cam, ha, hb, self._mutation, None if probe is None else probe.ctypes.data) == 0
                self.last_probe = probe
