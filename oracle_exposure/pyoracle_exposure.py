"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_exposure/liboracle_exposure.so: the CPU oracle (oracle/, unchanged) plus the exposure and tonemapping of
ST_OPT_TONEMAPPING / ST_OPT_AUTO_EXPOSURE (exposure.cpp).  `ExposureOracle` wraps any oracle engine (the plain one or one of its
extensions): it meters each rendered frame's `output` the way the device does and stores the Rgba8 frame through the display
transform.  Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle

_DIR = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_DIR), "oracle")
LIB = os.path.join(_DIR, "liboracle_exposure.so")
# the oracle's own flags (oracle/Makefile)
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
            "-Wno-misleading-indentation"]
OPT_TONEMAPPING, OPT_AUTO_EXPOSURE = 20, 21
MODE_BVH_HEATMAP = 5
FIELDS = ("ev", "compensation", "ev_min", "ev_max", "low", "high", "speed_up", "speed_down")
DEFAULTS = dict(ev=0.0, compensation=0.0, ev_min=-8.0, ev_max=8.0, low=0.1, high=0.9, speed_up=0.05, speed_down=1.0 / 60.0)
# deliberate mistakes (tests only): of the luminance, the bin centre, the window, the speeds, the order of exposure and T, the matrices
MUTATIONS = {"rec601": 1, "bin_lower_edge": 2, "no_window": 3, "swap_speeds": 4, "expose_after_t": 5, "aces_transposed": 6,
             "agx_row_major": 7, "agx_no_pow": 8}


def build(force=False):
    srcs = [os.path.join(_DIR, "exposure.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ORACLE, n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "exposure.cpp")])
    return LIB


_LIB = []


def lib():
    if not _LIB:
        build()
        mine = C.CDLL(LIB)
        F = np.ctypeslib.ndpointer(np.float32, flags="C")
        U = np.ctypeslib.ndpointer(np.uint32, flags="C")
        B = np.ctypeslib.ndpointer(np.uint8, flags="C")
        mine.orc_expo_histogram.argtypes, mine.orc_expo_histogram.restype = [F, C.c_long, U, C.c_int], C.c_int
        mine.orc_expo_meter.argtypes, mine.orc_expo_meter.restype = [U, U, F, C.c_int], C.c_int
        mine.orc_expo_display.argtypes, mine.orc_expo_display.restype = [F, C.c_long, C.c_int, C.c_float, C.c_float, B, C.c_int], C.c_int
        mine.orc_expo_transform.argtypes, mine.orc_expo_transform.restype = [F, C.c_long, C.c_int, F, C.c_int], C.c_int
        mine.orc_expo_log2.argtypes, mine.orc_expo_log2.restype = [F, F, C.c_long], None
        mine.orc_expo_pow.argtypes, mine.orc_expo_pow.restype = [C.c_float, C.c_float], C.c_float
        _LIB.append(mine)
    return _LIB[0]


def _mut(mutation):
    return MUTATIONS[mutation] if mutation else 0


def _frame(output):
    return np.ascontiguousarray(np.asarray(output, np.float32).reshape(-1))


def params(**fields):
    """st_exposure's 8 floats (float32) from keyword fields over the defaults."""
    v = dict(DEFAULTS, **fields)
    return np.array([v[n] for n in FIELDS], np.float32)


def histogram(output, mutation=None):
    """The 256 bin counts of a frame's `output` (any shape with 4 floats per pixel)."""
    o = _frame(output)
    bins = np.zeros(256, np.uint32)
    lib().orc_expo_histogram(o, o.size // 4, bins, _mut(mutation))
    return bins


def meter(bins, state, p, mutation=None):
    """One frame's metering and adaptation: returns the new state (5 uint32 words: ev, target bits, counted, kept, frames)."""
    s = np.array(state, np.uint32).copy()
    lib().orc_expo_meter(np.ascontiguousarray(bins, np.uint32), s, np.ascontiguousarray(p, np.float32), _mut(mutation))
    return s


def display(output, op, ev=0.0, compensation=0.0, mutation=None):
    """The Rgba8 store of a frame's `output`: op 0 today's, 1..4 through exposure 2^(compensation - ev) and T.  Returns n x 4 bytes."""
    o = _frame(output)
    out = np.zeros(o.size, np.uint8)
    lib().orc_expo_display(o, o.size // 4, int(op), np.float32(ev), np.float32(compensation), out, _mut(mutation))
    return out.reshape(-1, 4)


def transform(x, op, mutation=None):
    """T(x) in float32 (x: n x 3)."""
    a = np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1))
    out = np.zeros_like(a)
    lib().orc_expo_transform(a, a.size // 3, int(op), out, _mut(mutation))
    return out.reshape(-1, 3)


def log2_x(a):
    a = np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1))
    out = np.zeros_like(a)
    lib().orc_expo_log2(a, out, a.size)
    return out


def pow_det(x, y):
    return np.float32(lib().orc_expo_pow(float(x), float(y)))


def state_ev(state):
    return np.asarray(state, np.uint32)[0:1].view(np.float32)[0]


class ExposureOracle:
    """An oracle engine with ST_OPT_TONEMAPPING, ST_OPT_AUTO_EXPOSURE and st_set_exposure, which take effect at the next tick as on the
    device.  Every other verb goes to the wrapped engine.  `rgba8(cam)` is what st_copy_output(ST_FORMAT_RGBA8_SRGB) stores;
    `read_buffer(cam, "exposure")` the metering state.  `mutation` (tests only) applies one deliberate mistake, see MUTATIONS."""

    def __init__(self, engine, mutation=None):
        self.engine = engine
        self.mutation = mutation
        self.tonemapping, self.auto_exposure, self.exposure = 0, False, params()
        self._pending = (0, False, params())
        self._desc, self._state, self._bins = {}, {}, {}

    def __getattr__(self, name):
        return getattr(self.engine, name)

    def set_option(self, option, value):
        t, a, p = self._pending
        if option == OPT_TONEMAPPING:
            assert 0 <= value <= 4
            self._pending = (int(value), a, p)
        elif option == OPT_AUTO_EXPOSURE:
            assert value in (0, 1)
            self._pending = (t, bool(value), p)
        else:
            self.engine.set_option(option, value)

    def set_exposure(self, **fields):
        t, a, _ = self._pending
        self._pending = (t, a, params(**fields))

    def create_camera(self, mode, denoise, ref_depth, w, h, transform16, projection16):
        cam = self.engine.create_camera(mode, denoise, ref_depth, w, h, transform16, projection16)
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h)
        return cam

    def update_camera(self, cam, mode, denoise, ref_depth, w, h, transform16, projection16):
        if self._desc[cam] != (mode, bool(denoise), ref_depth, w, h):
            self._state.pop(cam, None)   # camera reallocation: the next metering is a first frame
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h)
        self.engine.update_camera(cam, mode, denoise, ref_depth, w, h, transform16, projection16)

    def _metering(self):
        return self.tonemapping != 0 and self.auto_exposure

    def meters(self, cam):
        return self._metering() and self._desc[cam][0] != MODE_BVH_HEATMAP

    def tick(self):
        self.engine.tick()
        was = self._metering()
        self.tonemapping, self.auto_exposure, self.exposure = self._pending
        if was != self._metering():
            self._state.clear()

    def render_camera(self, cam):
        self.engine.render_camera(cam)
        if self.meters(cam):
            self.meter_output(cam, self.engine.read_buffer(cam, "output"))

    def meter_output(self, cam, output):
        """Meters `output` as the camera's frame (what the device's metering step does after the composition)."""
        bins = histogram(output, self.mutation)
        self._state[cam] = meter(bins, self._state.get(cam, np.zeros(5, np.uint32)), self.exposure, self.mutation)
        self._bins[cam] = bins

    def ev(self, cam):
        return state_ev(self._state[cam]) if self.meters(cam) else np.float32(self.exposure[0])

    def rgba8(self, cam, output=None):
        """The Rgba8 frame (h x w x 4 bytes) of the camera's `output` (or of the given one)."""
        w, h = self._desc[cam][3], self._desc[cam][4]
        o = self.engine.read_buffer(cam, "output") if output is None else output
        op = 0 if self._desc[cam][0] == MODE_BVH_HEATMAP else self.tonemapping
        if self.meters(cam) and cam not in self._state:
            self._state[cam] = np.zeros(5, np.uint32)
        return display(o, op, self.ev(cam), self.exposure[1], self.mutation).reshape(h, w, 4)

    def read_buffer(self, cam, name):
        if name == "exposure":
            if not self.meters(cam) or cam not in self._state:
                raise KeyError(name)
            words = np.concatenate([self._state[cam], self._bins.get(cam, np.zeros(256, np.uint32)).astype(np.uint32)])
            return words.view(np.float32)
        return self.engine.read_buffer(cam, name)
