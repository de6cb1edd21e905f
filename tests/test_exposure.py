"""Exposure and tonemapping (ST_OPT_TONEMAPPING, ST_OPT_AUTO_EXPOSURE, st_set_exposure): the oracle extension against known answers
written from the rule, against the float64 restatement (with its deliberate mistakes) and against today's store with the options off;
the CUDA path against the extension (strict tier bit for bit), its lifetime and isolation, and the strip entry points."""
import math
import os
import re

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle import pyoracle
from oracle_envmap import pyoracle_envmap as EM
from oracle_exposure import pyoracle_exposure as X
from tests import ref64_exposure as R
from tests import ref64_svgf as RS

OPT_TONEMAPPING, OPT_AUTO_EXPOSURE, STAT_EXPOSURE_METERINGS = 20, 21, 15
OPT_FUSED_PASSES, OPT_TEMPORAL_AA = 11, 18
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = (1, 2, 3, 4)
GREY = 0.3   # L = 0.3: log2 L = -1.737, bin 114 (y = 114.10, clear of both edges)


def _empty_sky(w, h, c=GREY, intensity=1.0):
    """An empty scene in Reference mode under a constant environment map c, the sun below the horizon: every pixel is c * intensity."""
    return dict(name="empty_sky", meshes={}, materials={}, instances=[], lights=[], sun=(0.0, -1.2),
                camera=dict(mode=scenes.MODE_REFERENCE, denoise=False, ref_depth=1, w=w, h=h, transform=_eye(0),
                            projection=scenes.perspective_infinite_reverse_rh(math.pi / 3.0, w / h, 0.1)),
                environment_map=dict(rgba=np.full((4, 8, 4), c, np.float32), intensity=intensity, rotation=0.0))


def _eye(f):
    """A camera that moves every frame (Reference mode restarts its accumulation), always seeing the constant sky."""
    return scenes.look_at_transform((0.05 * f, 1.0, 0.0), (0.05 * f, 1.0, -1.0))


def _u32(words):
    return np.asarray(words, np.float32).view(np.uint32)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_constants_agree_across_header_python_and_rust():
    from strolle_b200 import engine as E
    header = open(os.path.join(ROOT, "include", "strolle_b200.h")).read()
    rust = open(os.path.join(ROOT, "rust", "strolle-b200-sys", "src", "lib.rs")).read()
    for name, value in (("OPT_TONEMAPPING", 20), ("OPT_AUTO_EXPOSURE", 21), ("STAT_EXPOSURE_METERINGS", 15)):
        assert re.search(rf"ST_{name} = {value}\b", header), name
        assert f"pub const ST_{name}: c_int = {value};" in rust, name
        assert getattr(E, name) == value and getattr(X, name, value) == value
    assert "pub fn st_set_exposure(e: *mut st_engine, exposure: *const st_exposure) -> c_int;" in rust
    assert "pub fn st_multi_set_exposure(m: *mut st_multi, exposure: *const st_exposure) -> c_int;" in rust
    assert list(E.EXPOSURE_DEFAULTS) == list(X.FIELDS) and E.EXPOSURE_DEFAULTS == X.DEFAULTS


def test_primitive_bounds():
    """The measured errors of the flag-independent primitives stay inside the bounds the float64 restatement uses: log2_x against
    log2, pow_det(2, y) over the EV range, pow_det(u, 2.2) over AgX's output range."""
    rng = np.random.RandomState(3)
    x = np.concatenate([2.0 ** rng.uniform(-40, 40, 200000), rng.uniform(0.5, 2.0, 100000)]).astype(np.float32)
    err = np.abs(X.log2_x(x).astype(np.float64) - np.log2(x.astype(np.float64)))
    assert (err <= R.LOG2_ABS * (1 + np.abs(np.log2(x.astype(np.float64))))).all(), err.max()
    for y in np.concatenate([np.linspace(-24, 24, 2001), rng.uniform(-24, 24, 2000)]).astype(np.float32):
        got = float(X.pow_det(2.0, y))
        assert abs(got - 2.0 ** float(y)) <= 2.0 ** float(y) * R.POW2_REL(float(y)), y
    for u in np.concatenate([np.linspace(1e-6, 2.0, 4001), 2.0 ** rng.uniform(-20, 1, 2000)]).astype(np.float32):
        got, want = float(X.pow_det(u, 2.2)), float(u) ** float(np.float32(2.2))
        assert abs(got - want) <= want * R.POW22_REL(float(u)), u


def test_known_answers_of_the_operators():
    """Reinhard of luminance 1 gives 1/2; ACES of 0 stores 0; exposure only is today's store of 2^(comp - ev) x; each operator's byte
    on a grey ramp matches float64 wherever float64 decides it."""
    one = np.array([[1.0, 1.0, 1.0, 1.0]], np.float32)
    assert np.allclose(X.transform(one[:, :3], 2), 0.5, rtol=0, atol=0)
    half = X.display(np.array([[0.5, 0.5, 0.5, 1.0]], np.float32), 0)
    assert (X.display(one, 2) == half).all()
    assert (X.display(np.zeros((1, 4), np.float32), 3)[0, :3] == 0).all()
    assert (X.display(np.array([[0.25, 0.25, 0.25, 1]], np.float32), 1, ev=-1.0) == half).all()   # 0.25 x 2^(0 - (-1)) = 0.5
    ramp = np.zeros((4096, 4), np.float32)
    ramp[:, :3] = (2.0 ** np.linspace(-12, 8, 4096))[:, None]
    for op in OPS:
        got = X.display(ramp, op, ev=0.5, compensation=0.25)[:, :3].astype(np.int64)
        lo, hi = R.display(ramp, op, 0.5, 0.25)
        assert ((got >= lo) & (got <= hi)).all(), op
        assert (lo == hi).mean() > 0.95, op


def test_options_off_keep_todays_store(blue_noise):
    """Op 0 is k_output_rgba8's store: on the plain oracle's Cornell frame it equals ref64_svgf's float64 sRGB store byte for byte
    outside that store's own rounding window."""
    sc = scenes.cornell(64, 36)
    eo = pyoracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(eo, sc)
    eo.tick(); eo.render_camera(cam)
    out = eo.read_buffer(cam, "output").reshape(-1, 4)
    got = X.display(out, 0)[:, :3].reshape(-1).astype(np.int64)
    want, t, dt = RS.srgb_encode(out[:, :3].reshape(-1))
    near = np.abs(t - np.round(t)) <= dt
    assert ((got == want) | (near & (np.abs(got - want) <= 1))).all()
    assert (X.display(out, 0)[:, 3] == 255).all()


def _sky_oracle(blue_noise, w=16, h=8, mutation=None):
    eo = X.ExposureOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise), mutation=mutation)
    sc = _empty_sky(w, h)
    return eo, scenes.apply(eo, sc), sc


def _sky_frame(eo, cam, sc, f, intensity=1.0):
    c = sc["camera"]
    eo.set_environment_map(rgba=sc["environment_map"]["rgba"], intensity=intensity)
    eo.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], c["w"], c["h"], _eye(f), c["projection"])
    eo.tick(); eo.render_camera(cam)


def test_constant_sky_meters_one_bin(blue_noise):
    """Under a constant sky c every pixel is c: one histogram bin, EV = that bin's centre - log2 0.18 (clamped), and each operator's
    byte is the float64 one."""
    eo, cam, sc = _sky_oracle(blue_noise)
    for op in OPS:
        eo.set_option(OPT_TONEMAPPING, op); eo.set_option(OPT_AUTO_EXPOSURE, 1)
        _sky_frame(eo, cam, sc, op)
        out = eo.read_buffer(cam, "output").reshape(-1, 4)
        assert np.allclose(out[:, :3], GREY, rtol=1e-6)
        words = _u32(eo.read_buffer(cam, "exposure"))
        assert words[5 + 114] == 128 and words[5:261].sum() == 128 and words[2] == 128
        ev = np.float32(-16.0 + 114.5 / 8.0 - math.log2(0.18))
        assert words[0:1].view(np.float32)[0] == ev and words[1:2].view(np.float32)[0] == ev
        rgba = eo.rgba8(cam).reshape(-1, 4)[:, :3].astype(np.int64)
        lo, hi = R.display(out, op, ev, 0.0)
        assert ((rgba >= lo) & (rgba <= hi)).all() and (lo == hi).all(), op
    eo.set_exposure(ev_min=-8.0, ev_max=0.5)   # clamped
    _sky_frame(eo, cam, sc, 9)
    assert _u32(eo.read_buffer(cam, "exposure"))[1:2].view(np.float32)[0] == np.float32(0.5)


def test_intensity_step_moves_the_ev_by_the_speeds(blue_noise):
    """Eight times the sky's intensity moves the target up three stops; the EV climbs by exactly speed_up per frame and lands on the
    target; back to one, it falls by speed_down per frame and lands."""
    eo, cam, sc = _sky_oracle(blue_noise)
    eo.set_option(OPT_TONEMAPPING, 4); eo.set_option(OPT_AUTO_EXPOSURE, 1)
    eo.set_exposure(speed_up=0.5, speed_down=0.25)
    base = np.float32(-16.0 + 114.5 / 8.0 - math.log2(0.18))
    _sky_frame(eo, cam, sc, 0)
    ev = X.state_ev(_u32(eo.read_buffer(cam, "exposure")))
    assert ev == base
    high = np.float32(-16.0 + (114.5 + 24) / 8.0 - math.log2(0.18))
    for target, speed, intensity in ((high, np.float32(0.5), 8.0), (base, np.float32(-0.25), 1.0)):
        f = 1
        while True:
            _sky_frame(eo, cam, sc, f, intensity)
            words = _u32(eo.read_buffer(cam, "exposure"))
            assert words[1:2].view(np.float32)[0] == target
            new = words[0:1].view(np.float32)[0]
            want = target if abs(float(target) - float(ev)) <= abs(float(speed)) else np.float32(ev + speed)
            assert new == want, (f, new, want)
            ev = new
            f += 1
            if ev == target:
                break
        assert f > 3


def test_window_cuts_inside_a_bin():
    """low / high windows that cut inside a bin keep only that bin's overlap: the extension's EV is the rule's, written by hand."""
    p = X.params(low=0.25, high=0.625)   # both exact in f32
    counts = np.zeros(256, np.uint32)
    counts[100], counts[110], counts[120] = 30, 50, 20   # N = 100: window [25, ceil(62.5)) keeps 5 of bin 100 and 33 of bin 110
    s = X.meter(counts, np.zeros(5, np.uint32), p)
    c = lambda b: -16.0 + (b + 0.5) / 8.0
    want = np.float32((5 * c(100) + 33 * c(110)) / 38 - math.log2(0.18))
    assert X.state_ev(s) == want and s[2] == 100 and s[3] == 38
    assert R.meter(counts, p, (0.0, 0))[0] == want


MOTION = {"cornell": None, "dungeon": None, "env_sunlit": None, "env_courtyard": scenes.env_courtyard_motion}


def _scene_frames(name, blue_noise, w=48, h=27, frames=13):
    """The oracle's `output` over 13 moving frames (the camera drifts, or orbits in env_courtyard)."""
    sc = {"cornell": scenes.cornell, "dungeon": scenes.dungeon, "env_sunlit": scenes.env_sunlit, "env_courtyard": scenes.env_courtyard}[name](w, h)
    eo = EM.EnvMapOracleEngine(blue_noise=blue_noise) if "environment_map" in sc else pyoracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(eo, sc)
    c = sc["camera"]
    outs = []
    for f in range(frames):
        if MOTION[name]:
            xf, _ = MOTION[name](f)
        else:
            t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
            t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
            xf = t.reshape(-1)
        eo.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
        eo.tick(); eo.render_camera(cam)
        outs.append(eo.read_buffer(cam, "output").reshape(-1, 4).copy())
    return outs


def _violations(outs, op, auto, mutation=None):
    """Runs the extension (with `mutation`) over the frames and counts where it leaves the float64 restatement's bound."""
    p = X.params(ev=-1.5, compensation=0.5)
    state = np.zeros(5, np.uint32)
    bad = 0
    for out in outs:
        ev = np.float32(p[0])
        if auto:
            counts = X.histogram(out, mutation)
            lo, hi = R.bins(out)
            bad += R.check_histogram(counts, lo, hi)
            want = R.meter(counts, p, (X.state_ev(state), state[4]))
            state = X.meter(counts, state, p, mutation)
            bad += int(X.state_ev(state) != want[0])
            ev = X.state_ev(state)
        got = X.display(out, op, ev, p[1], mutation)[:, :3].astype(np.int64)
        blo, bhi = R.display(out, op, ev, p[1])
        bad += int(((got < blo) | (got > bhi)).sum())
    return bad


@pytest.fixture(scope="module")
def scene_frames(blue_noise):
    return {n: _scene_frames(n, blue_noise) for n in MOTION}


@pytest.mark.parametrize("name", list(MOTION))
def test_extension_inside_the_float64_bound(scene_frames, name):
    """On cornell, dungeon, env_sunlit and env_courtyard over 13 moving frames, for every operator with auto exposure on and off, the
    extension's bins, EV and bytes lie inside the float64 restatement's bound."""
    for op in OPS:
        for auto in (False, True):
            assert _violations(scene_frames[name], op, auto) == 0, (name, op, auto)


@pytest.mark.parametrize("mutation,op", [("rec601", 2), ("bin_lower_edge", 1), ("no_window", 1), ("swap_speeds", 1), ("expose_after_t", 4),
                                         ("aces_transposed", 3), ("agx_row_major", 4), ("agx_no_pow", 4)])
def test_deliberate_mistakes_leave_the_bound(scene_frames, mutation, op):
    """Each deliberate mistake, run through the same frames with auto exposure on, leaves the float64 bound somewhere."""
    assert sum(_violations(scene_frames[n], op, True, mutation) for n in ("env_sunlit", "env_courtyard", "cornell")) > 0


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu_engine(blue_noise, exact=True, fused=False, opts=None):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    if exact and fused:
        e.set_option(OPT_FUSED_PASSES, 1)
    for k, v in (opts or {}).items():
        e.set_option(k, v)
    return e


def _rgba8(e, cam, w, h):
    from strolle_b200.engine import FORMAT_RGBA8_SRGB
    out = np.zeros((h, w, 4), np.uint8)
    e.copy_output(cam, out, FORMAT_RGBA8_SRGB)
    return out


INVALID = (dict(ev=math.inf), dict(ev=math.nan), dict(compensation=-math.inf), dict(compensation=math.nan), dict(ev_min=math.nan),
           dict(ev_max=math.inf), dict(ev_min=2.0, ev_max=1.0), dict(low=math.nan), dict(high=math.nan), dict(low=0.5, high=0.5),
           dict(low=0.9, high=0.1), dict(low=-0.1), dict(high=1.5), dict(speed_up=-1.0), dict(speed_down=-0.25), dict(speed_up=math.nan),
           dict(speed_down=math.inf))


@pytest.mark.gpu
def test_gpu_invalid_options_and_settings(blue_noise):
    """Option values outside their range and every out-of-range st_exposure field are refused on a live engine; a refused call changes
    nothing: an engine that received every refused call renders the same bytes and exposure words, frame for frame, as one that never
    did (manual EV, then metered)."""
    import strolle_b200
    for opt, bad in ((OPT_TONEMAPPING, -1), (OPT_TONEMAPPING, 5), (OPT_AUTO_EXPOSURE, 2), (OPT_AUTO_EXPOSURE, -1)):
        with pytest.raises(strolle_b200.StrolleError):
            _gpu_engine(blue_noise).set_option(opt, bad)
    sc = scenes.env_courtyard(96, 54)
    a, b = _gpu_engine(blue_noise), _gpu_engine(blue_noise)
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    for e in (a, b):
        e.set_option(OPT_TONEMAPPING, 4); e.set_exposure(ev=-1.25, compensation=0.5, speed_up=0.3)
    for f in range(6):
        if f == 3:
            for e in (a, b):
                e.set_option(OPT_AUTO_EXPOSURE, 1)
        for fields in INVALID:
            with pytest.raises(strolle_b200.StrolleError, match="st_set_exposure"):
                a.set_exposure(**fields)
        with pytest.raises(strolle_b200.StrolleError):
            a.set_option(OPT_TONEMAPPING, 7)
        a.tick(); b.tick(); a.render_camera(ca); b.render_camera(cb)
        assert (_rgba8(a, ca, 96, 54) == _rgba8(b, cb, 96, 54)).all(), f"frame {f}"
        if f >= 3:
            assert (_u32(a.read_buffer(ca, "exposure")) == _u32(b.read_buffer(cb, "exposure"))).all(), f"frame {f}"
    assert X.state_ev(_u32(a.read_buffer(ca, "exposure"))) != np.float32(-1.25)


@pytest.mark.gpu
def test_gpu_group_invalid_settings_change_nothing(blue_noise):
    """st_multi_set_exposure refuses every out-of-range field as a whole and changes no member: a two-strip group that received every
    refused call still matches the single-GPU frame (which never did) bit for bit with its fixed exposure."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA8_SRGB
    w, h = 256, 288
    sc = scenes.cornell(w, h)
    one = strolle_b200.Engine(blue_noise=blue_noise)
    grp = strolle_b200.MultiEngine([0, 0], blue_noise=blue_noise)
    c1, cn = scenes.apply(one, sc), scenes.apply(grp, sc)
    for e in (one, grp):
        e.set_option(OPT_TONEMAPPING, 3); e.set_exposure(ev=0.75, compensation=-0.25)
    for f in range(3):
        for fields in INVALID:
            with pytest.raises(strolle_b200.StrolleError, match="st_set_exposure"):
                grp.set_exposure(**fields)
        one.tick(); grp.tick()
        x, y = np.zeros((h, w, 4), np.uint8), np.zeros((h, w, 4), np.uint8)
        one.render_camera(c1, x, FORMAT_RGBA8_SRGB); grp.render_camera(cn, y, FORMAT_RGBA8_SRGB)
        assert (x == y).all(), f"frame {f}"


def _moving(sc, f):
    c = sc["camera"]
    if sc["name"] == "env_courtyard":
        return scenes.env_courtyard_motion(f)[0]
    t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
    t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
    return t.reshape(-1)


def _run_pair(blue_noise, sc, op, auto, frames=13, fused=False, taa=False, end_to_end=False):
    """The device and the extension over `frames` moving frames with a brightness step at frame 6 (the map's intensity x 8, or the
    exposure compensation where the scene has no map); returns the number of frames compared."""
    w, h = sc["camera"]["w"], sc["camera"]["h"]
    e = _gpu_engine(blue_noise, fused=fused, opts={OPT_TONEMAPPING: op, OPT_AUTO_EXPOSURE: int(auto), OPT_TEMPORAL_AA: int(taa)})
    x = X.ExposureOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    x.set_option(OPT_TONEMAPPING, op); x.set_option(OPT_AUTO_EXPOSURE, int(auto))
    cg = scenes.apply(e, sc)
    cx = scenes.apply(x, sc) if end_to_end else x.create_camera(sc["camera"]["mode"], sc["camera"]["denoise"], sc["camera"]["ref_depth"], w, h,
                                                              sc["camera"]["transform"], sc["camera"]["projection"])
    c = sc["camera"]
    for f in range(frames):
        step = f >= 6
        if "environment_map" in sc:
            m = sc["environment_map"]
            e.set_environment_map(rgba=m["rgba"], intensity=m["intensity"] * (8.0 if step else 1.0))
            if end_to_end:
                x.set_environment_map(rgba=m["rgba"], intensity=m["intensity"] * (8.0 if step else 1.0))
        for eng, cam in ((e, cg), (x, cx)):
            eng.set_exposure(compensation=1.0 if step else 0.0, ev=-0.5, speed_up=0.2, speed_down=0.1)
            if end_to_end or eng is e:
                eng.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, _moving(sc, f), c["projection"])
        e.tick()
        if end_to_end:
            x.tick(); x.render_camera(cx)
            out = x.read_buffer(cx, "output")
        else:
            x.tick()   # the wrapped engine renders nothing: the extension meters the device's own frame
        e.render_camera(cg)
        dev_out = e.read_buffer(cg, "output")
        if end_to_end:
            assert (dev_out.view(np.uint32) == out.view(np.uint32)).all(), f"frame {f}: output"
        elif x.meters(cx):
            x.meter_output(cx, dev_out)
        got = _rgba8(e, cg, w, h)
        want = x.rgba8(cx, dev_out)
        assert (got == want).all(), f"frame {f}: {int((got != want).any(-1).sum())} pixels differ"
        if auto:
            gw, xw = _u32(e.read_buffer(cg, "exposure")), _u32(x.read_buffer(cx, "exposure"))
            assert (gw == xw).all(), f"frame {f}: exposure words {np.nonzero(gw != xw)[0][:8]}"
    return frames


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("auto", [False, True], ids=["manual", "auto"])
def test_gpu_strict_bit_exact(blue_noise, op, auto):
    """Strict tier: the Rgba8 frame and the exposure words (EV bits and all 256 counts) equal the extension's over 13 moving frames with
    a brightness step, at 224x126 (unfused) and 67x45 (fused), on env_courtyard."""
    _run_pair(blue_noise, scenes.env_courtyard(224, 126), op, auto)
    _run_pair(blue_noise, scenes.env_courtyard(67, 45), op, auto, fused=True)


@pytest.mark.gpu
def test_gpu_strict_end_to_end_and_modes(blue_noise):
    """End to end against the extension over its own oracle frames (Cornell-like env scene at 67x45), Reference mode, and temporal AA on
    (metering the resolved `output`)."""
    _run_pair(blue_noise, scenes.env_courtyard(67, 45), 4, True, frames=4, end_to_end=True)
    _run_pair(blue_noise, scenes.env_courtyard(67, 45, mode=scenes.MODE_REFERENCE), 3, True)
    _run_pair(blue_noise, scenes.env_sunlit(67, 45), 2, True, taa=True)


def _decode(rgba):
    """Rgba8UnormSrgb bytes (h, w, 4) to linear RGB floats (n, 3)."""
    c = np.asarray(rgba, np.float64)[..., :3].reshape(-1, 3) / 255.0
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


@pytest.mark.gpu
@pytest.mark.parametrize("op", [2, 4])
def test_gpu_product_tier(blue_noise, op):
    """Product tier (the default fast-math kernels) against the extension run end to end on the oracle, auto exposure on, 9 moving
    frames of env_courtyard with a brightness step: the G-buffer stays bit-exact; the decoded Rgba8 frame stays within
    max(1e-3, 1.5 x the option-off drift) relative per-channel L2 of the extension's, the option-off drift being the same measure
    between today's store of the two `output` frames; the EV stays within 0.02 of the extension's.  The display and metering kernels
    are also exact on the product frame itself: its bytes and exposure words equal the extension's run on that frame."""
    from tests.util import rel_l2
    w, h = 160, 90
    sc = scenes.env_courtyard(w, h)
    e = _gpu_engine(blue_noise, exact=False, opts={OPT_TONEMAPPING: op, OPT_AUTO_EXPOSURE: 1})
    x = X.ExposureOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))   # end to end: the oracle renders, the extension meters and stores
    own = X.ExposureOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))   # the extension over the device's own frame
    cg, cx = scenes.apply(e, sc), scenes.apply(x, sc)
    co = own.create_camera(sc["camera"]["mode"], True, 1, w, h, sc["camera"]["transform"], sc["camera"]["projection"])
    for eng in (x, own):
        eng.set_option(OPT_TONEMAPPING, op); eng.set_option(OPT_AUTO_EXPOSURE, 1)
    c, m = sc["camera"], sc["environment_map"]
    worst = 0.0
    for f in range(9):
        xf = scenes.env_courtyard_motion(f)[0]
        for eng, cam in ((e, cg), (x, cx)):
            eng.set_environment_map(rgba=m["rgba"], intensity=m["intensity"] * (4.0 if f >= 5 else 1.0))
            eng.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
            eng.tick()
        own.tick()
        e.render_camera(cg); x.render_camera(cx)
        for name in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b"):
            assert (e.read_buffer(cg, name).view(np.uint32) == x.read_buffer(cx, name).view(np.uint32)).all(), f"frame {f}: {name}"
        dev_out, ora_out = e.read_buffer(cg, "output"), x.read_buffer(cx, "output")
        own.meter_output(co, dev_out)
        got = _rgba8(e, cg, w, h)
        assert (got == own.rgba8(co, dev_out)).all(), f"frame {f}: the display kernel on the product frame"
        assert (_u32(e.read_buffer(cg, "exposure")) == _u32(own.read_buffer(co, "exposure"))).all(), f"frame {f}: metering on the product frame"
        on, want = _decode(got), _decode(x.rgba8(cx))
        off_dev, off_ora = _decode(X.display(dev_out, 0)), _decode(X.display(ora_out, 0))
        for ch in range(3):
            drift = rel_l2(off_dev[:, ch], off_ora[:, ch])
            err = rel_l2(on[:, ch], want[:, ch])
            worst = max(worst, err)
            assert err <= max(1e-3, 1.5 * drift), f"frame {f} channel {ch}: {err:.2e} against option-off drift {drift:.2e}"
        ev_dev, ev_ext = X.state_ev(_u32(e.read_buffer(cg, "exposure"))), x.ev(cx)
        assert abs(float(ev_dev) - float(ev_ext)) <= 0.02, (f, ev_dev, ev_ext)
    print(f"product tier op {op}: worst decoded rel L2 {worst:.2e}")


@pytest.mark.gpu
def test_gpu_lifetime_and_isolation(blue_noise):
    """The Rgba32F frame and `output` do not change with the options; two copies do not adapt twice; the heat map keeps today's store;
    the metering counter counts; the state is freed when metering turns off and restarts when it turns on or the camera is reallocated;
    two cameras adapt independently."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA32F
    w, h = 96, 54
    sc = scenes.env_sunlit(w, h)
    a, b = _gpu_engine(blue_noise, exact=False), _gpu_engine(blue_noise, exact=False, opts={OPT_TONEMAPPING: 3, OPT_AUTO_EXPOSURE: 1})
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    c = sc["camera"]
    c2 = b.create_camera(c["mode"], c["denoise"], c["ref_depth"], w, h, scenes.look_at_transform((0.0, 0.5, 4.0), (0.0, 30.0, -10.0)), c["projection"])
    for f in range(4):
        a.tick(); b.tick()
        a.render_camera(ca); b.render_camera(cb); b.render_camera(c2)
        fa, fb = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 4), np.float32)
        a.copy_output(ca, fa, FORMAT_RGBA32F); b.copy_output(cb, fb, FORMAT_RGBA32F)
        assert (fa.view(np.uint32) == fb.view(np.uint32)).all()
        assert (a.read_buffer(ca, "output").view(np.uint32) == b.read_buffer(cb, "output").view(np.uint32)).all()
    w1 = _u32(b.read_buffer(cb, "exposure"))
    _rgba8(b, cb, w, h); _rgba8(b, cb, w, h)
    assert (_u32(b.read_buffer(cb, "exposure")) == w1).all() and w1[4] == 4
    assert X.state_ev(w1) != X.state_ev(_u32(b.read_buffer(c2, "exposure")))   # the camera looking at the sky meters differently
    assert b.get_stat(STAT_EXPOSURE_METERINGS) == 8
    b.set_option(OPT_AUTO_EXPOSURE, 0); b.tick(); b.render_camera(cb)
    with pytest.raises(strolle_b200.StrolleError):
        b.read_buffer(cb, "exposure")
    assert b.get_stat(STAT_EXPOSURE_METERINGS) == 8
    b.set_option(OPT_AUTO_EXPOSURE, 1); b.tick(); b.render_camera(cb)
    assert _u32(b.read_buffer(cb, "exposure"))[4] == 1
    b.update_camera(cb, c["mode"], c["denoise"], c["ref_depth"], w + 2, h, c["transform"], c["projection"])
    b.tick(); b.render_camera(cb)
    assert _u32(b.read_buffer(cb, "exposure"))[4] == 1
    # heat map: today's bytes with the options on
    for eng in (a, b):
        cam = eng.create_camera(scenes.MODE_BVH_HEATMAP, False, 1, w, h, c["transform"], c["projection"])
        eng.tick(); eng.render_camera(cam)
        eng._hm = _rgba8(eng, cam, w, h)
    assert (a._hm == b._hm).all()


@pytest.mark.gpu
@pytest.mark.parametrize("members", [2, 3])
def test_gpu_strips_fixed_exposure_and_auto_refused(blue_noise, members):
    """Two- and three-strip groups on one device match the single-GPU Rgba8 frame bit for bit with a fixed exposure; auto exposure on a
    group returns ST_ERR_INVALID, and the group renders once it is off."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA8_SRGB
    w, h = 256, 288
    sc = scenes.cornell(w, h)
    one = strolle_b200.Engine(blue_noise=blue_noise)
    grp = strolle_b200.MultiEngine([0] * members, blue_noise=blue_noise)
    c1, cn = scenes.apply(one, sc), scenes.apply(grp, sc)
    for eng in (one, grp):
        eng.set_option(OPT_TONEMAPPING, 4); eng.set_exposure(ev=-1.0, compensation=0.5)
    for f in range(3):
        one.tick(); grp.tick()
        a, b = np.zeros((h, w, 4), np.uint8), np.zeros((h, w, 4), np.uint8)
        one.render_camera(c1, a, FORMAT_RGBA8_SRGB); grp.render_camera(cn, b, FORMAT_RGBA8_SRGB)
        assert (a == b).all(), f"frame {f}"
    grp.set_option(OPT_AUTO_EXPOSURE, 1); grp.tick()
    with pytest.raises(Exception, match="AUTO_EXPOSURE"):
        grp.render_camera(cn, b, FORMAT_RGBA8_SRGB)
    grp.set_option(OPT_AUTO_EXPOSURE, 0); grp.tick()
    grp.render_camera(cn, b, FORMAT_RGBA8_SRGB)


@pytest.mark.gpu
def test_gpu_tonemapped_strips_on_real_gpus():
    """On a box with >= 2 GPUs: tools/verify_multigpu_exposure.py under torchrun (one process per GPU) — the tonemapped store with a
    fixed exposure through both gathers of st_render_strips is the single-GPU frame, and auto exposure is refused.  Skipped on
    single-GPU boxes."""
    import socket
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tools", "verify_multigpu_exposure.py")],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [l for l in p.stdout.splitlines() if l.startswith(("OK", "FAIL"))]
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert len(lines) == 4 and all(l.startswith("OK") for l in lines), "\n".join(lines)
