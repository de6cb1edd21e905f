"""ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle_dof/liboracle_dof.so: the CPU oracle (oracle/, unchanged) plus the depth of field of
ST_OPT_DEPTH_OF_FIELD (dof.cpp).  `DofOracle` wraps any oracle engine (the plain one or one of its extensions) in a `BloomOracle`
(and so an `ExposureOracle`): it defocuses each rendered frame the way the device does, after the composition and before the metering
and the pyramid, and hands the defocused frame to them and to the Rgba8 store.  Imported only by tests/ and tools/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_exposure import pyoracle_exposure as X
from oracle_bloom import pyoracle_bloom as B

_DIR = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_DIR)
LIB = os.path.join(_DIR, "liboracle_dof.so")
OPT_DEPTH_OF_FIELD, STAT_DEPTH_OF_FIELD_GATHERS = 23, 17
MODE_BVH_HEATMAP, MODE_REFERENCE = 5, 6
FIELDS = ("focal_distance", "aperture_f_stops", "sensor_height", "max_radius")
DEFAULTS = dict(focal_distance=10.0, aperture_f_stops=1.0, sensor_height=0.01866, max_radius=16.0)
HEADER_WORDS, TILE, MAX_RADIUS, TAPS = 16, 16, 32, 81
# deliberate mistakes (tests only)
MUTATIONS = {"coc_sign": 1, "ray_distance": 2, "no_background_limit": 3, "no_density": 4, "no_dilation": 5, "offsets_truncated": 6,
             "sky_in_focus": 7, "nan_kept": 8, "lens_shading_stream": 9}


def build(force=False):
    srcs = [os.path.join(_DIR, "dof.cpp"), os.path.abspath(__file__)] + \
           [os.path.join(_ROOT, "oracle", n) for n in ("oracle.cpp", "orc_math.hpp", "orc_gpu.hpp", "orc_passes.hpp", "orc_host.hpp")]
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++"] + X.CXXFLAGS + ["-o", LIB, os.path.join(_DIR, "dof.cpp")])
    return LIB


_LIB = []


def lib():
    if not _LIB:
        build()
        mine = C.CDLL(LIB)
        F = np.ctypeslib.ndpointer(np.float32, flags="C")
        I = np.ctypeslib.ndpointer(np.int32, flags="C")
        mine.orc_dof_taps.argtypes, mine.orc_dof_taps.restype = [I, F, C.c_int], C.c_int
        mine.orc_dof_consts.argtypes, mine.orc_dof_consts.restype = [F, F, F, C.c_int, F], C.c_int
        mine.orc_dof_run.argtypes = [F, F, F, C.c_int, C.c_int, F, F, F, F, F, C.c_int]
        mine.orc_dof_run.restype = C.c_int
        mine.orc_dof_rays.argtypes, mine.orc_dof_rays.restype = [F, C.c_int, C.c_int, F], C.c_int
        mine.orc_dof_lens.argtypes, mine.orc_dof_lens.restype = [F, F, F, F], C.c_int
        mine.orc_dof_lens_rays.argtypes, mine.orc_dof_lens_rays.restype = [F, C.c_int, C.c_int, F, C.c_uint32, F, F], C.c_int
        mine.orc_dof_render_reference.argtypes, mine.orc_dof_render_reference.restype = [C.c_void_p, C.c_int, F, C.c_int], C.c_int
        _LIB.append(mine)
    return _LIB[0]


def _mut(mutation):
    return MUTATIONS[mutation] if mutation else 0


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1))


def params(**fields):
    """st_depth_of_field as a dict over the defaults."""
    unknown = set(fields) - set(DEFAULTS)
    assert not unknown, unknown
    return dict(DEFAULTS, **fields)


def _lens(p):
    return np.array([p[n] for n in FIELDS], np.float32)


def taps(mutation=None):
    """The tap table: (32 x 81 x 2) integer offsets and (32 x 81) float32 distances."""
    dxy, d = np.zeros(2 * MAX_RADIUS * TAPS, np.int32), np.zeros(MAX_RADIUS * TAPS, np.float32)
    lib().orc_dof_taps(dxy, d, _mut(mutation))
    return dxy.reshape(MAX_RADIUS, TAPS, 2), d.reshape(MAX_RADIUS, TAPS)


def consts(p, transform16, projection16, h):
    """(defocused, float32 {f, A, k, F, R, forward.xyz}) of a frame."""
    out = np.zeros(8, np.float32)
    active = lib().orc_dof_consts(_lens(p), _f32(transform16), _f32(projection16), int(h), out)
    return bool(active), out


def rays(camera40, w, h):
    """The frame's camera ray directions (h x w x 3 float32), the oracle's camera_ray."""
    out = np.zeros(w * h * 3, np.float32)
    lib().orc_dof_rays(_f32(camera40), int(w), int(h), out)
    return out.reshape(h, w, 3)


def lens(p, transform16, projection16):
    """(a lens, float32 {h, F, right.xyz, up.xyz, fwd.xyz}): Reference mode's thin lens of a camera."""
    out = np.zeros(11, np.float32)
    on = lib().orc_dof_lens(_lens(p), _f32(transform16), _f32(projection16), out)
    return bool(on), out


def lens_rays(camera40, w, h, L, seed):
    """The thin-lens primary rays (origins, directions; h x w x 3 float32 each) of lens L (lens()) with lens dispatch seed `seed`."""
    o, d = np.zeros(w * h * 3, np.float32), np.zeros(w * h * 3, np.float32)
    lib().orc_dof_lens_rays(_f32(camera40), int(w), int(h), _f32(L), int(seed) & 0xffffffff, o, d)
    return o.reshape(h, w, 3), d.reshape(h, w, 3)


def dispatch_seed(base, frame, k):
    """engine.cu dispatch_seed: the seed of dispatch k of a frame."""
    m = 0xffffffff
    s = (base ^ ((frame * 64 + k) & m)) & m
    s = (s * 747796405 + 2891336453) & m
    w = (((s >> ((s >> 28) + 4)) ^ s) * 277803737) & m
    return (w >> 22) ^ w


LENS_DISPATCH = 27   # K_LENS (engine.cu)


def render_reference(engine, cam, p, mutation=None):
    """Renders a Reference-mode frame of an oracle engine (procedural sky) with K1 / K2's depth-0 rays leaving the thin lens of p;
    returns whether the lens applied (F > f: otherwise the engine rendered through the pinhole)."""
    return bool(lib().orc_dof_render_reference(engine.h, int(cam), _lens(p), _mut(mutation)))


def run(output, t, camera40, w, h, p, transform16, projection16, mutation=None):
    """The "depth_of_field" words (float32 view) and the defocused frame (h x w x 4) of a frame's `output` with primary hit distances t."""
    tiles = ((w + TILE - 1) // TILE) * ((h + TILE - 1) // TILE)
    words = np.zeros(HEADER_WORDS + w * h + tiles, np.float32)
    frame = np.zeros(w * h * 4, np.float32)
    lib().orc_dof_run(_f32(output), _f32(t), _f32(camera40), int(w), int(h), _lens(p), _f32(transform16), _f32(projection16), words, frame,
                      _mut(mutation))
    return words, frame.reshape(h, w, 4)


class _Defocused:
    """The wrapped engine as the exposure and bloom extensions see it: its `output` is the defocused frame while the camera is
    defocused."""

    def __init__(self, engine, owner):
        self.engine, self.owner = engine, owner

    def __getattr__(self, name):
        return getattr(self.engine, name)

    def render_camera(self, cam):
        if self.owner.lens_on(cam):
            render_reference(self.engine, cam, self.owner.p, self.owner.mutation)
            return
        self.engine.render_camera(cam)
        if self.owner.defocuses(cam):
            self.owner.defocus(cam)

    def read_buffer(self, cam, name):
        if name == "output" and self.owner.defocuses(cam) and cam in self.owner._frame:
            return self.owner._frame[cam].reshape(-1)
        return self.engine.read_buffer(cam, name)


class DofOracle:
    """An oracle engine with ST_OPT_DEPTH_OF_FIELD and st_set_depth_of_field (and, through the wrapped BloomOracle, bloom, exposure and
    tonemapping), which take effect at the next tick as on the device.  `frame(cam)` is what st_copy_output(ST_FORMAT_RGBA32F) stores,
    `rgba8(cam)` what st_copy_output(ST_FORMAT_RGBA8_SRGB) stores; `read_buffer(cam, "depth_of_field")` the words and
    `read_buffer(cam, "output")` the sharp frame.  `mutation` (tests only) applies one deliberate mistake, see MUTATIONS."""

    def __init__(self, engine, mutation=None):
        self.base = engine
        self.b = B.BloomOracle(X.ExposureOracle(_Defocused(engine, self)))
        self.mutation = mutation
        self.dof, self.p = False, params()
        self._pending = (False, params())
        self._desc, self._frame, self._words = {}, {}, {}
        self.gathers = 0

    def __getattr__(self, name):
        return getattr(self.b, name)

    def set_option(self, option, value):
        if option == OPT_DEPTH_OF_FIELD:
            assert value in (0, 1)
            self._pending = (bool(value), self._pending[1])
        else:
            self.b.set_option(option, value)

    def set_depth_of_field(self, **fields):
        self._pending = (self._pending[0], params(**fields))

    def create_camera(self, mode, denoise, ref_depth, w, h, transform16, projection16):
        cam = self.b.create_camera(mode, denoise, ref_depth, w, h, transform16, projection16)
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h, np.asarray(transform16, np.float32), np.asarray(projection16, np.float32))
        return cam

    def update_camera(self, cam, mode, denoise, ref_depth, w, h, transform16, projection16):
        if self._desc[cam][:5] != (mode, bool(denoise), ref_depth, w, h):
            self._frame.pop(cam, None); self._words.pop(cam, None)   # camera reallocation
        self._desc[cam] = (mode, bool(denoise), ref_depth, w, h, np.asarray(transform16, np.float32), np.asarray(projection16, np.float32))
        self.b.update_camera(cam, mode, denoise, ref_depth, w, h, transform16, projection16)

    def defocuses(self, cam):
        return self.dof and self._desc[cam][0] not in (MODE_BVH_HEATMAP, MODE_REFERENCE)

    def lens_on(self, cam):
        """Reference mode samples the lens in its primary rays (restated with the procedural sky)."""
        return self.dof and self._desc[cam][0] == MODE_REFERENCE

    def tick(self):
        self.b.tick()
        was = self.dof
        self.dof, self.p = self._pending
        if was != self.dof:
            self._frame.clear(); self._words.clear()

    def depth(self, cam):
        """The primary hit distances of the frame last rendered (the current G-buffer's depth)."""
        frame = int(self.base.lib.orc_frame(self.base.h)) - 1   # the wrapped engine's frame, as its last tick gave it to the cameras
        name = "prim_gbuffer_d0_b" if frame % 2 == 1 else "prim_gbuffer_d0_a"
        w, h = self._desc[cam][3], self._desc[cam][4]
        return self.base.read_buffer(cam, name).reshape(h, w, 4)[..., 0]

    def defocus(self, cam, output=None, t=None, camera40=None):
        """Defocuses `output` (the camera's sharp frame by default) with hit distances t and the frame's camera, as the device's pass."""
        mode, _, _, w, h, xf, pr = self._desc[cam]
        o = self.base.read_buffer(cam, "output") if output is None else output
        t = self.depth(cam) if t is None else t
        c40 = self.base.read_buffer(cam, "curr_camera") if camera40 is None else camera40
        self._words[cam], self._frame[cam] = run(o, t, c40, w, h, self.p, xf, pr, self.mutation)
        self.gathers += 1
        return self._words[cam], self._frame[cam]

    def frame(self, cam):
        """The Rgba32F frame (h x w x 4)."""
        w, h = self._desc[cam][3], self._desc[cam][4]
        if self.defocuses(cam):
            return self._frame.get(cam, np.zeros((h, w, 4), np.float32))
        return self.base.read_buffer(cam, "output").reshape(h, w, 4)

    def read_buffer(self, cam, name):
        if name == "depth_of_field":
            if not self.defocuses(cam) or cam not in self._words:
                raise KeyError(name)
            return self._words[cam]
        if name == "output":
            return self.base.read_buffer(cam, name)
        return self.b.read_buffer(cam, name)
