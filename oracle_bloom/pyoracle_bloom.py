"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_bloom/liboracle_bloom.so: the CPU oracle (oracle/, unchanged) with the exposure extension
(oracle_exposure/) plus the bloom of ST_OPT_BLOOM (bloom.cpp).  `BloomOracle` wraps any oracle engine (the plain one or one of its
extensions) in an `ExposureOracle`: it builds each rendered frame's pyramid the way the device does, after the metering, and stores the
Rgba8 frame with the glow composited.  Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_exposure import pyoracle_exposure as X

_DIR = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_DIR)
LIB = os.path.join(_DIR, "liboracle_bloom.so")
OPT_BLOOM, STAT_BLOOM_PYRAMIDS = 22, 16
MODE_BVH_HEATMAP = X.MODE_BVH_HEATMAP
FIELDS = ("intensity", "scatter", "threshold", "softness", "levels", "mode")
DEFAULTS = dict(intensity=0.15, scatter=0.7, threshold=0.0, softness=0.0, levels=7, mode=0)
HEADER_WORDS = 20
# deliberate mistakes (tests only)
MUTATIONS = {"karis_all": 1, "karis_none": 2, "tent_111": 3, "sizes_round_up": 4, "wrap_edges": 5, "swap_scatter": 6, "expose_after": 7,
             "prefilter_after_karis": 8, "swap_modes": 9, "nan_not_cleared": 10}


def build(force=False):
    srcs = [os.path.join(_DIR, "bloom.cpp"), os.path.abspath(__file__), os.path.join(_ROOT, "oracle_exposure", "exposure.cpp")] + \
           [os.path.join(_ROOT, "oracle", n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + X.CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "bloom.cpp")])
    return LIB


_LIB = []


def lib():
    if not _LIB:
        build()
        mine = C.CDLL(LIB)
        F = np.ctypeslib.ndpointer(np.float32, flags="C")
        B = np.ctypeslib.ndpointer(np.uint8, flags="C")
        mine.orc_bloom_pyramid.argtypes = [F, C.c_int, C.c_int, C.c_float, F, C.c_int, C.c_int, F, C.c_long, C.c_int]
        mine.orc_bloom_pyramid.restype = C.c_long
        mine.orc_bloom_store.argtypes = [F, C.c_int, C.c_int, C.c_int, C.c_float, F, C.c_int, F, B, C.c_int]
        mine.orc_bloom_store.restype = C.c_int
        _LIB.append(mine)
    return _LIB[0]


def _mut(mutation):
    return MUTATIONS[mutation] if mutation else 0


def params(**fields):
    """st_bloom as a dict over the defaults."""
    unknown = set(fields) - set(DEFAULTS)
    assert not unknown, unknown
    return dict(DEFAULTS, **fields)


def _floats(p):
    return np.array([p["intensity"], p["scatter"], p["threshold"], p["softness"]], np.float32)


def exposure_scale(tonemapping, ev, compensation):
    """The pyramid's and the store's exposure s: pow_det(2, compensation - ev) with tonemapping on, 1 off."""
    if tonemapping == 0:
        return np.float32(1.0)
    return X.pow_det(2.0, np.float32(np.float32(compensation) - np.float32(ev)))


def pyramid(output, w, h, s, p, mutation=None):
    """st_read_buffer("bloom") words (float32 view) of a frame's `output` (h x w x 4 floats) with exposure s."""
    o = np.ascontiguousarray(np.asarray(output, np.float32).reshape(-1))
    if mutation == "expose_after":
        s = 1.0
    f = _floats(p)
    n = lib().orc_bloom_pyramid(o, w, h, np.float32(s), f, int(p["levels"]), int(p["mode"]), np.zeros(1, np.float32), 0, _mut(mutation))
    words = np.zeros(n, np.float32)
    lib().orc_bloom_pyramid(o, w, h, np.float32(s), f, int(p["levels"]), int(p["mode"]), words, n, _mut(mutation))
    return words


def store(output, w, h, op, s, p, words, mutation=None):
    """The Rgba8 store (h x w x 4 bytes) of `output` with the glow of `words`."""
    o = np.ascontiguousarray(np.asarray(output, np.float32).reshape(-1))
    out = np.zeros(w * h * 4, np.uint8)
    lib().orc_bloom_store(o, w, h, int(op), np.float32(s), _floats(p), int(p["mode"]), np.ascontiguousarray(words, np.float32), out, _mut(mutation))
    return out.reshape(h, w, 4)


def empty_pyramid(w, h, levels):
    """The zero-filled pyramid of a camera that has not built one yet."""
    z = np.zeros((h, w, 4), np.float32)
    return pyramid(z, w, h, 1.0, params(levels=levels))


class BloomOracle:
    """An oracle engine with ST_OPT_BLOOM and st_set_bloom (and, through the wrapped ExposureOracle, ST_OPT_TONEMAPPING,
    ST_OPT_AUTO_EXPOSURE and st_set_exposure), which take effect at the next tick as on the device.  `rgba8(cam)` is what
    st_copy_output(ST_FORMAT_RGBA8_SRGB) stores; `read_buffer(cam, "bloom")` the pyramid.  `mutation` (tests only) applies one deliberate
    mistake, see MUTATIONS."""

    def __init__(self, engine, mutation=None):
        self.x = engine if isinstance(engine, X.ExposureOracle) else X.ExposureOracle(engine)
        self.mutation = mutation
        self.bloom, self.p = False, params()
        self._pending = (False, params())
        self._pyr = {}
        self.pyramids = 0

    def __getattr__(self, name):
        return getattr(self.x, name)

    def set_option(self, option, value):
        if option == OPT_BLOOM:
            assert value in (0, 1)
            self._pending = (bool(value), self._pending[1])
        else:
            self.x.set_option(option, value)

    def set_bloom(self, **fields):
        self._pending = (self._pending[0], params(**fields))

    def create_camera(self, mode, denoise, ref_depth, w, h, transform16, projection16):
        return self.x.create_camera(mode, denoise, ref_depth, w, h, transform16, projection16)

    def update_camera(self, cam, mode, denoise, ref_depth, w, h, transform16, projection16):
        if self.x._desc[cam] != (mode, bool(denoise), ref_depth, w, h):
            self._pyr.pop(cam, None)   # camera reallocation: the pyramid starts zeroed
        self.x.update_camera(cam, mode, denoise, ref_depth, w, h, transform16, projection16)

    def blooms(self, cam):
        return self.bloom and self.x._desc[cam][0] != MODE_BVH_HEATMAP

    def tick(self):
        self.x.tick()
        was, levels = self.bloom, self.p["levels"]
        self.bloom, self.p = self._pending
        if was != self.bloom or levels != self.p["levels"]:
            self._pyr.clear()

    def render_camera(self, cam):
        self.x.render_camera(cam)
        if self.blooms(cam):
            self.build_pyramid(cam, self.x.engine.read_buffer(cam, "output"))

    def _scale(self, cam):
        return exposure_scale(self.x.tonemapping, self.x.ev(cam), self.x.exposure[1])

    def build_pyramid(self, cam, output):
        """Builds the pyramid of `output` as the camera's frame (what the device's pyramid step does after the metering)."""
        w, h = self.x._desc[cam][3], self.x._desc[cam][4]
        self._pyr[cam] = pyramid(output, w, h, self._scale(cam), self.p, self.mutation)
        self.pyramids += 1

    def _words(self, cam):
        w, h = self.x._desc[cam][3], self.x._desc[cam][4]
        if cam not in self._pyr:
            self._pyr[cam] = empty_pyramid(w, h, self.p["levels"])
        return self._pyr[cam]

    def rgba8(self, cam, output=None):
        """The Rgba8 frame (h x w x 4 bytes) of the camera's `output` (or of the given one)."""
        if not self.blooms(cam):
            return self.x.rgba8(cam, output)
        w, h = self.x._desc[cam][3], self.x._desc[cam][4]
        o = self.x.engine.read_buffer(cam, "output") if output is None else output
        if self.x.meters(cam) and cam not in self.x._state:
            self.x._state[cam] = np.zeros(5, np.uint32)
        return store(o, w, h, self.x.tonemapping, self._scale(cam), self.p, self._words(cam), self.mutation)

    def read_buffer(self, cam, name):
        if name == "bloom":
            if not self.blooms(cam):
                raise KeyError(name)
            return self._words(cam)
        return self.x.read_buffer(cam, name)
