"""Bloom (ST_OPT_BLOOM, st_set_bloom): the oracle extension against known answers written from the rule, against the float64
restatement (with its deliberate mistakes) and against today's store; the CUDA path against the extension (strict tier bit for bit,
product tier within the option-off drift), its refusals, lifetime and isolation, and the strip entry points."""
import math
import os
import re

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle import pyoracle
from oracle_envmap import pyoracle_envmap as EM
from oracle_exposure import pyoracle_exposure as X
from oracle_bloom import pyoracle_bloom as B
from tests import ref64_bloom as RB

OPT_TONEMAPPING, OPT_AUTO_EXPOSURE, OPT_BLOOM, STAT_BLOOM_PYRAMIDS = 20, 21, 22, 16
OPT_FUSED_PASSES, OPT_TEMPORAL_AA = 11, 18
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _u32(words):
    return np.asarray(words, np.float32).view(np.uint32)


def _levels(words):
    from strolle_b200.engine import parse_bloom
    return parse_bloom(words)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_constants_agree_across_header_python_and_rust():
    from strolle_b200 import engine as E
    header = open(os.path.join(ROOT, "include", "strolle_b200.h")).read()
    rust = open(os.path.join(ROOT, "rust", "strolle-b200-sys", "src", "lib.rs")).read()
    for name, value in (("OPT_BLOOM", 22), ("STAT_BLOOM_PYRAMIDS", 16)):
        assert re.search(rf"ST_{name} = {value}\b", header), name
        assert f"pub const ST_{name}: c_int = {value};" in rust, name
        assert getattr(E, name) == value and getattr(B, name) == value
    assert "pub fn st_set_bloom(e: *mut st_engine, bloom: *const st_bloom) -> c_int;" in rust
    assert "pub fn st_multi_set_bloom(m: *mut st_multi, bloom: *const st_bloom) -> c_int;" in rust
    assert "pub struct st_bloom" in rust
    assert list(E.BLOOM_DEFAULTS) == list(B.FIELDS) and E.BLOOM_DEFAULTS == B.DEFAULTS
    assert re.search(r"NULL restores the defaults \{0\.15, 0\.7, 0, 0, 7, 0\}", header)
    hl = open(os.path.join(ROOT, "rust", "strolle-b200", "src", "lib.rs")).read()
    assert "pub fn set_bloom(&mut self, bloom: Option<&Bloom>)" in hl and "pub enum BloomMode" in hl


def _const(w, h, c):
    o = np.zeros((h, w, 4), np.float32)
    o[..., :3] = c
    o[..., 3] = 1.0
    return o


@pytest.mark.parametrize("levels", [7, 1, 8])
def test_constant_frame_stays_constant(levels):
    """A constant frame: every level equals the constant within the float64 bound, and with mode 0 the Rgba8 bytes equal the bloom-off
    bytes wherever float64 decides them (tonemapping off and AgX)."""
    w, h = 45, 29
    c = np.array([0.3, 0.7, 1.9], np.float32)
    o = _const(w, h, c)
    p = B.params(levels=levels, intensity=0.6, scatter=0.45)
    words = B.pyramid(o, w, h, 1.0, p)
    lo, hi, down, up = RB.display(o, w, h, 0, 0, 0.0, 0.0, p)
    assert RB.check_words(words, down, up) == 0
    lv = _levels(words)
    for arr in lv["down"] + lv["up"]:
        assert np.allclose(arr, c, rtol=8 * 2.0 ** -23, atol=0), arr
    for op, tm in ((0, 0), (4, 1)):
        s = B.exposure_scale(tm, 0.5, 0.0)
        got = B.store(o, w, h, op, s, p, B.pyramid(o, w, h, s, p)).reshape(-1, 4)[:, :3].astype(np.int64)
        off = X.display(o, op, 0.5, 0.0)[:, :3].astype(np.int64)
        lo, hi, _, _ = RB.display(o, w, h, op, tm, 0.5, 0.0, p)
        decided = lo == hi
        assert ((got >= lo) & (got <= hi)).all()
        assert (got[decided] == off[decided]).all() and decided.mean() > 0.5, op


def test_threshold_above_the_brightest_pixel_adds_nothing():
    """With the threshold above the frame's brightest exposed value, mode 1 stores exactly the bloom-off bytes."""
    w, h = 40, 24
    o = (np.random.RandomState(5).rand(h, w, 4) * 3.0).astype(np.float32)
    p = B.params(threshold=4.0, softness=0.0, mode=1, intensity=2.5)
    for op, tm in ((0, 0), (2, 1), (4, 1)):
        s = B.exposure_scale(tm, 0.0, 0.0)
        words = B.pyramid(o, w, h, s, p)
        assert (_u32(words)[20:] == 0).all()
        assert (B.store(o, w, h, op, s, p, words).reshape(-1, 4) == X.display(o, op)).all(), op


def test_nan_inf_and_negative_pixels_do_not_spread():
    """A NaN, an inf and a negative pixel give the same pyramid bits as 0 at that pixel."""
    w, h = 31, 19
    o = (np.random.RandomState(6).rand(h, w, 4)).astype(np.float32)
    zero = o.copy()
    zero[3, 4, :3] = 0.0
    zero[10, 20, :3] = 0.0
    zero[15, 7, 1] = 0.0
    bad = o.copy()
    bad[3, 4, :3] = np.nan
    bad[10, 20, :3] = np.inf
    bad[15, 7, 1] = -5.0
    for p in (B.params(), B.params(threshold=0.5, softness=0.5)):
        a, b = B.pyramid(bad, w, h, 1.0, p), B.pyramid(zero, w, h, 1.0, p)
        assert (_u32(a) == _u32(b)).all()
        assert (_u32(B.pyramid(bad, w, h, 1.0, p, "nan_not_cleared")) != _u32(b)).any()


def test_single_bright_pixel_glow_energy_and_spread():
    """One pixel away from the edges: the glow B (up_0 brought to full resolution) holds the pixel's exposed energy (each level's filter
    weights sum to 1), within the float64 bound and the Karis weight of a dim pixel (1 - 1e-4); a bright pixel's energy is damped by its
    Karis weight (a firefly); larger scatter or more levels spread the glow further."""
    w, h = 256, 160
    tm, ev = 1, 1.0
    s = B.exposure_scale(tm, ev, 0.0)

    def glow(rgb, p):
        o = _const(w, h, 0.0)
        o[80, 129, :3] = rgb
        words = B.pyramid(o, w, h, s, p)
        _, _, down, up = RB.display(o, w, h, 1, tm, ev, 0.0, p)
        assert RB.check_words(words, down, up) == 0
        lv = _levels(words)
        Bf, dB = RB._tent(*up[0], w, h)
        Bx, _ = RB._tent(lv["up"][0].astype(np.float64), np.zeros_like(lv["up"][0], np.float64), w, h)
        assert (np.abs(Bx - Bf) <= dB + 4 * RB.U * Bf).all()
        return Bx, np.asarray(rgb, np.float64) * float(s)

    p = B.params(levels=4, scatter=0.5)
    Bx, x = glow((4e-4, 2e-4, 1e-4), p)
    assert np.allclose(Bx.sum(axis=(0, 1)), x, rtol=1e-4, atol=0), (Bx.sum(axis=(0, 1)), x)
    Bb, xb = glow((400.0, 200.0, 100.0), p)
    assert (Bb.sum(axis=(0, 1)) < 0.5 * xb).all()
    yy, xx = np.mgrid[0:h, 0:w]
    r2 = lambda g: float((g.sum(-1) * ((yy - 80) ** 2 + (xx - 129) ** 2)).sum() / g.sum())
    base = r2(Bx)
    assert r2(glow((4e-4, 2e-4, 1e-4), B.params(levels=4, scatter=0.9))[0]) > base
    assert r2(glow((4e-4, 2e-4, 1e-4), B.params(levels=6, scatter=0.5))[0]) > base
    assert r2(glow((4e-4, 2e-4, 1e-4), B.params(levels=2, scatter=0.5))[0]) < base


@pytest.mark.parametrize("w,h", [(1, 37), (41, 1), (1, 1), (3, 2)])
def test_one_pixel_wide_and_high_frames(w, h):
    """1-pixel-wide and -high frames: every level is 1 texel on the short side, and the bound holds, for L = 1 and L = 8."""
    o = (np.random.RandomState(w * 7 + h).rand(h, w, 4) * 2.0).astype(np.float32)
    for levels in (1, 8):
        p = B.params(levels=levels)
        words = B.pyramid(o, w, h, 1.0, p)
        lo, hi, down, up = RB.display(o, w, h, 0, 0, 0.0, 0.0, p)
        assert RB.check_words(words, down, up) == 0
        got = B.store(o, w, h, 0, 1.0, p, words).reshape(-1, 4)[:, :3]
        assert ((got >= lo) & (got <= hi)).all()
        assert [tuple(s) for s in _levels(words)["sizes"]] == [(max(1, w >> (k + 1)), max(1, h >> (k + 1))) for k in range(levels)]


SCENES = {"cornell": scenes.cornell, "dungeon": scenes.dungeon, "env_sunlit": scenes.env_sunlit, "aa_edges": scenes.aa_edges}


def _scene_frames(name, blue_noise, w=48, h=27, frames=13):
    """The oracle's `output` over 13 moving frames."""
    sc = SCENES[name](w, h)
    eo = EM.EnvMapOracleEngine(blue_noise=blue_noise) if "environment_map" in sc else pyoracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(eo, sc)
    c = sc["camera"]
    outs = []
    for f in range(frames):
        t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
        t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
        eo.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t.reshape(-1), c["projection"])
        eo.tick(); eo.render_camera(cam)
        outs.append(eo.read_buffer(cam, "output").reshape(h, w, 4).copy())
    return outs


CASES = [dict(op=0, auto=False, p=B.params()),
         dict(op=4, auto=False, p=B.params(mode=1, intensity=0.4, threshold=1.0, softness=0.5)),
         dict(op=4, auto=True, p=B.params(scatter=0.85, levels=8)),
         dict(op=0, auto=False, p=B.params(mode=1, intensity=1.5, threshold=0.25, softness=0.0, levels=4)),
         dict(op=2, auto=True, p=B.params(threshold=0.5, softness=1.0, levels=1))]


def _violations(outs, case, mutation=None):
    """Runs the extension (with `mutation`) over the frames, metering like the device when auto exposure is on, and counts the pyramid
    floats and bytes outside the float64 bound."""
    h, w = outs[0].shape[:2]
    xp = X.params(ev=-1.0, compensation=0.5)
    state = np.zeros(5, np.uint32)
    bad = 0
    op, p = case["op"], case["p"]
    tm = int(op != 0)
    for out in outs:
        ev = np.float32(xp[0])
        if case["auto"] and tm:
            state = X.meter(X.histogram(out), state, xp)
            ev = X.state_ev(state)
        s = B.exposure_scale(tm, ev, xp[1])
        words = B.pyramid(out, w, h, s, p, mutation)
        got = B.store(out, w, h, op, s, p, words, mutation).reshape(-1, 4)[:, :3].astype(np.int64)
        lo, hi, down, up = RB.display(out, w, h, op, tm, ev, xp[1], p)
        bad += RB.check_words(words, down, up) + int(((got < lo) | (got > hi)).sum())
    return bad


@pytest.fixture(scope="module")
def scene_frames(blue_noise):
    frames = {n: _scene_frames(n, blue_noise) for n in SCENES}
    frames["odd"] = _scene_frames("cornell", blue_noise, w=37, h=23, frames=4)
    return frames


@pytest.mark.parametrize("name", list(SCENES) + ["odd"])
def test_extension_inside_the_float64_bound(scene_frames, name):
    """On cornell, dungeon, env_sunlit and aa_edges over 13 moving frames (and an odd 37x23 size), for both modes, threshold 0 and a
    soft threshold, tonemapping 0 and on, auto exposure off and on, the extension's pyramid and bytes lie inside the float64 bound."""
    for case in CASES:
        assert _violations(scene_frames[name], case) == 0, (name, case)


@pytest.mark.parametrize("mutation,case", [("karis_all", 0), ("karis_none", 0), ("tent_111", 0), ("sizes_round_up", 0), ("wrap_edges", 0),
                                           ("swap_scatter", 2), ("expose_after", 2), ("prefilter_after_karis", 1), ("swap_modes", 3)])
def test_deliberate_mistakes_leave_the_bound(scene_frames, mutation, case):
    """Each deliberate mistake, run through the same frames, leaves the float64 bound somewhere."""
    assert sum(_violations(scene_frames[n][:4], CASES[case], mutation) for n in ("env_sunlit", "aa_edges", "odd")) > 0


def test_nan_not_cleared_leaves_the_bound(scene_frames):
    """The NaN mistake: a frame with one NaN pixel leaves the float64 bound (which clears it)."""
    out = scene_frames["aa_edges"][0].copy()
    out[10, 20, 1] = np.nan
    assert _violations([out], CASES[0], "nan_not_cleared") > 0
    assert _violations([out], CASES[0]) == 0


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


def _moving(sc, f):
    t = np.asarray(sc["camera"]["transform"], np.float32).reshape(4, 4).copy()
    t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
    return t.reshape(-1)


def _run_pair(blue_noise, sc, op, auto, bloom, frames=13, fused=False, taa=False):
    """The device and the extension (over the device's own `output`) over `frames` moving frames with a brightness step at frame 6 (the
    map's intensity x 8 or the compensation): the Rgba8 frame and the "bloom" words, bit for bit."""
    w, h = sc["camera"]["w"], sc["camera"]["h"]
    e = _gpu_engine(blue_noise, fused=fused, opts={OPT_TONEMAPPING: op, OPT_AUTO_EXPOSURE: int(auto), OPT_TEMPORAL_AA: int(taa), OPT_BLOOM: 1})
    x = B.BloomOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    for k, v in ((OPT_TONEMAPPING, op), (OPT_AUTO_EXPOSURE, int(auto)), (OPT_BLOOM, 1)):
        x.set_option(k, v)
    c = sc["camera"]
    cg = scenes.apply(e, sc)
    cx = x.create_camera(c["mode"], c["denoise"], c["ref_depth"], w, h, c["transform"], c["projection"])
    e.set_bloom(**bloom); x.set_bloom(**bloom)
    for f in range(frames):
        step = f >= 6
        if "environment_map" in sc:
            m = sc["environment_map"]
            e.set_environment_map(rgba=m["rgba"], intensity=m["intensity"] * (8.0 if step else 1.0))
        for eng in (e, x):
            eng.set_exposure(compensation=1.0 if step else 0.0, ev=-0.5, speed_up=0.2, speed_down=0.1)
        e.update_camera(cg, c["mode"], c["denoise"], c["ref_depth"], w, h, _moving(sc, f), c["projection"])
        e.tick(); x.tick()
        if f == 0:   # a copy before the first pyramid composites no glow from the zero-filled one
            _rgba8(e, cg, w, h)
            assert (_u32(e.read_buffer(cg, "bloom")) == _u32(x.read_buffer(cx, "bloom"))).all()
        e.render_camera(cg)
        dev_out = e.read_buffer(cg, "output")
        if x.x.meters(cx):
            x.x.meter_output(cx, dev_out)
        x.build_pyramid(cx, dev_out)
        gw, xw = _u32(e.read_buffer(cg, "bloom")), _u32(x.read_buffer(cx, "bloom"))
        assert gw.size == xw.size and (gw == xw).all(), f"frame {f}: {int((gw != xw).sum())} pyramid words differ"
        got = _rgba8(e, cg, w, h)
        want = x.rgba8(cx, dev_out)
        assert (got == want).all(), f"frame {f}: {int((got != want).any(-1).sum())} pixels differ"
    return frames


@pytest.mark.gpu
@pytest.mark.parametrize("op", [0, 1, 2, 3, 4])
def test_gpu_strict_bit_exact(blue_noise, op):
    """Strict tier: the Rgba8 frame and the "bloom" words equal the extension's over 13 moving frames, for every operator, auto exposure
    off then on, at 224x126 (unfused, energy-conserving, no threshold, L = 7) and 67x45 (fused, additive, a soft threshold, L = 8)."""
    _run_pair(blue_noise, scenes.env_courtyard(224, 126), op, False, B.params())
    _run_pair(blue_noise, scenes.env_sunlit(67, 45), op, op != 0, B.params(mode=1, intensity=0.7, threshold=1.0, softness=0.5, levels=8), fused=True)


@pytest.mark.gpu
def test_gpu_strict_levels_modes_and_taa(blue_noise):
    """L = 1 and L = 8 (one launch per level down to 1x1), Reference mode, temporal AA on, and aa_edges (an emissive quad and bar on
    black).  The one-launch tails of the tuning builds are checked against this build's words by tools/bloom_variants.py."""
    _run_pair(blue_noise, scenes.aa_edges(96, 64), 0, False, B.params(levels=1, intensity=0.5), frames=4)
    _run_pair(blue_noise, scenes.cornell(96, 64), 4, True, B.params(levels=8, scatter=0.95), frames=4)
    _run_pair(blue_noise, scenes.env_courtyard(67, 45, mode=scenes.MODE_REFERENCE), 3, True, B.params(), frames=4)
    _run_pair(blue_noise, scenes.env_sunlit(67, 45), 2, True, B.params(threshold=2.0), frames=4, taa=True)


def _decode(rgba):
    c = np.asarray(rgba, np.float64)[..., :3].reshape(-1, 3) / 255.0
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


@pytest.mark.gpu
@pytest.mark.parametrize("op", [0, 4])
def test_gpu_product_tier(blue_noise, op):
    """Product tier (the default fast-math kernels) against the extension run end to end on the oracle, 9 moving frames of env_sunlit:
    the G-buffer stays bit-exact; the decoded Rgba8 frame stays within max(1e-3, 1.5 x the option-off drift) relative per-channel L2;
    the pyramid and store kernels are exact on the product frame's own `output`."""
    from tests.util import rel_l2
    w, h = 160, 90
    sc = scenes.env_sunlit(w, h)
    opts = {OPT_TONEMAPPING: op, OPT_AUTO_EXPOSURE: int(op != 0), OPT_BLOOM: 1}
    e = _gpu_engine(blue_noise, exact=False, opts=opts)
    x = B.BloomOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    own = B.BloomOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    cg, cx = scenes.apply(e, sc), scenes.apply(x, sc)
    c = sc["camera"]
    co = own.create_camera(c["mode"], True, 1, w, h, c["transform"], c["projection"])
    for eng in (x, own):
        for k, v in opts.items():
            eng.set_option(k, v)
    for f in range(9):
        xf = _moving(sc, f)
        for eng, cam in ((e, cg), (x, cx)):
            eng.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
            eng.tick()
        own.tick()
        e.render_camera(cg); x.render_camera(cx)
        for name in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b"):
            assert (e.read_buffer(cg, name).view(np.uint32) == x.read_buffer(cx, name).view(np.uint32)).all(), f"frame {f}: {name}"
        dev_out, ora_out = e.read_buffer(cg, "output"), x.read_buffer(cx, "output")
        if own.x.meters(co):
            own.x.meter_output(co, dev_out)
        own.build_pyramid(co, dev_out)
        assert (_u32(e.read_buffer(cg, "bloom")) == _u32(own.read_buffer(co, "bloom"))).all(), f"frame {f}: pyramid on the product frame"
        got = _rgba8(e, cg, w, h)
        assert (got == own.rgba8(co, dev_out)).all(), f"frame {f}: the store on the product frame"
        on, want = _decode(got), _decode(x.rgba8(cx))
        off_dev, off_ora = _decode(X.display(dev_out, 0)), _decode(X.display(ora_out, 0))
        for ch in range(3):
            drift, err = rel_l2(off_dev[:, ch], off_ora[:, ch]), rel_l2(on[:, ch], want[:, ch])
            assert err <= max(1e-3, 1.5 * drift), f"frame {f} channel {ch}: {err:.2e} against option-off drift {drift:.2e}"


INVALID = (dict(intensity=math.nan), dict(scatter=math.inf), dict(threshold=-math.inf), dict(softness=math.nan), dict(mode=2), dict(mode=-1),
           dict(intensity=1.5), dict(intensity=-0.1), dict(intensity=-0.5, mode=1), dict(scatter=-0.01), dict(scatter=1.01),
           dict(softness=-0.5), dict(softness=2.0), dict(threshold=-1.0), dict(levels=0), dict(levels=9))


@pytest.mark.gpu
def test_gpu_refusals_change_nothing(blue_noise):
    """Option values outside 0..1 and every out-of-range st_bloom field are refused, on an engine and on a group; an engine that received
    every refused call renders the same bytes and pyramid, frame for frame, as one that never did."""
    import strolle_b200
    for bad in (-1, 2):
        with pytest.raises(strolle_b200.StrolleError):
            _gpu_engine(blue_noise).set_option(OPT_BLOOM, bad)
    w, h = 96, 54
    sc = scenes.env_sunlit(w, h)
    a, b = _gpu_engine(blue_noise, opts={OPT_BLOOM: 1, OPT_TONEMAPPING: 4}), _gpu_engine(blue_noise, opts={OPT_BLOOM: 1, OPT_TONEMAPPING: 4})
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    for e in (a, b):
        e.set_bloom(intensity=0.3, levels=5, threshold=0.5, softness=0.5)
    for f in range(3):
        for fields in INVALID:
            with pytest.raises(strolle_b200.StrolleError, match="st_set_bloom"):
                a.set_bloom(**fields)
        with pytest.raises(strolle_b200.StrolleError):
            a.set_option(OPT_BLOOM, 3)
        a.tick(); b.tick(); a.render_camera(ca); b.render_camera(cb)
        assert (_rgba8(a, ca, w, h) == _rgba8(b, cb, w, h)).all(), f"frame {f}"
        assert (_u32(a.read_buffer(ca, "bloom")) == _u32(b.read_buffer(cb, "bloom"))).all(), f"frame {f}"
    grp = strolle_b200.MultiEngine([0, 0], blue_noise=blue_noise)
    for fields in INVALID:
        with pytest.raises(strolle_b200.StrolleError, match="st_set_bloom"):
            grp.set_bloom(**fields)
    grp.set_bloom(mode=1, intensity=3.0)
    grp.set_bloom()


@pytest.mark.gpu
def test_gpu_option_off_and_linear_frames_unchanged(blue_noise):
    """The Rgba32F frame and `output` do not change with bloom on; an engine whose option was turned on and off again stores today's
    Rgba8 bytes (those of an engine that never bloomed), and frees the pyramid."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA32F
    w, h = 96, 54
    sc = scenes.aa_edges(w, h)
    a, b = _gpu_engine(blue_noise), _gpu_engine(blue_noise, opts={OPT_BLOOM: 1})
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    for f in range(5):
        if f == 3:
            b.set_option(OPT_BLOOM, 0)
        a.tick(); b.tick(); a.render_camera(ca); b.render_camera(cb)
        fa, fb = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 4), np.float32)
        a.copy_output(ca, fa, FORMAT_RGBA32F); b.copy_output(cb, fb, FORMAT_RGBA32F)
        assert (fa.view(np.uint32) == fb.view(np.uint32)).all()
        assert (a.read_buffer(ca, "output").view(np.uint32) == b.read_buffer(cb, "output").view(np.uint32)).all()
        same = (_rgba8(a, ca, w, h) == _rgba8(b, cb, w, h)).all()
        assert same == (f >= 3), f"frame {f}"
    with pytest.raises(strolle_b200.StrolleError):
        b.read_buffer(cb, "bloom")


@pytest.mark.gpu
def test_gpu_lifetime_isolation_heatmap_and_statistic(blue_noise):
    """One pyramid per rendered frame and none per st_copy_output; a copy before the first render composites no glow; the pyramid
    restarts zeroed after a resize and when `levels` changes; two cameras of different sizes do not interfere; the heat map is not
    bloomed."""
    import strolle_b200
    w, h = 96, 54
    sc = scenes.aa_edges(w, h)
    e = _gpu_engine(blue_noise, opts={OPT_BLOOM: 1})
    ref = _gpu_engine(blue_noise)
    c, cr = scenes.apply(e, sc), scenes.apply(ref, sc)
    k = sc["camera"]
    c2 = e.create_camera(k["mode"], k["denoise"], k["ref_depth"], 61, 37, k["transform"], k["projection"])
    e.tick(); ref.tick()
    with pytest.raises(strolle_b200.StrolleError):
        e.read_buffer(c, "bloom")   # allocated by the first render or copy
    _rgba8(e, c, w, h)
    assert (_u32(e.read_buffer(c, "bloom"))[20:] == 0).all()
    e.render_camera(c); ref.render_camera(cr)
    assert e.get_stat(STAT_BLOOM_PYRAMIDS) == 1
    first = _u32(e.read_buffer(c, "bloom")).copy()
    _rgba8(e, c, w, h); _rgba8(e, c, w, h)
    assert e.get_stat(STAT_BLOOM_PYRAMIDS) == 1
    e.render_camera(c2)
    assert e.get_stat(STAT_BLOOM_PYRAMIDS) == 2
    assert (_u32(e.read_buffer(c, "bloom")) == first).all()   # the second camera's pyramid is its own
    x = B.BloomOracle(pyoracle.OracleEngine(blue_noise=blue_noise))
    x.set_option(OPT_BLOOM, 1); x.tick()
    cx2 = x.create_camera(k["mode"], k["denoise"], k["ref_depth"], 61, 37, k["transform"], k["projection"])
    x.build_pyramid(cx2, e.read_buffer(c2, "output"))
    assert (_u32(e.read_buffer(c2, "bloom")) == _u32(x.read_buffer(cx2, "bloom"))).all()
    e.update_camera(c, k["mode"], k["denoise"], k["ref_depth"], w + 2, h, k["transform"], k["projection"])
    e.tick(); _rgba8(e, c, w + 2, h)
    words = _u32(e.read_buffer(c, "bloom"))
    assert words[1] == (w + 2) >> 1 and (words[20:] == 0).all()
    e.render_camera(c)
    assert (_u32(e.read_buffer(c, "bloom"))[20:] != 0).any()
    e.set_bloom(levels=3); e.tick(); _rgba8(e, c, w + 2, h)
    words = _u32(e.read_buffer(c, "bloom"))
    assert words[0] == 3 and (words[20:] == 0).all()
    hm = [eng.create_camera(scenes.MODE_BVH_HEATMAP, False, 1, w, h, k["transform"], k["projection"]) for eng in (e, ref)]
    e.tick(); ref.tick()
    e.render_camera(hm[0]); ref.render_camera(hm[1])
    assert (_rgba8(e, hm[0], w, h) == _rgba8(ref, hm[1], w, h)).all()
    with pytest.raises(strolle_b200.StrolleError):
        e.read_buffer(hm[0], "bloom")
    # a blooming camera switched to the heat map at the same size returns no pyramid
    e.render_camera(c2)
    assert _u32(e.read_buffer(c2, "bloom")).size > 20
    e.update_camera(c2, scenes.MODE_BVH_HEATMAP, False, 1, 61, 37, k["transform"], k["projection"])
    e.tick()
    with pytest.raises(strolle_b200.StrolleError):
        e.read_buffer(c2, "bloom")


@pytest.mark.gpu
def test_gpu_strips_refused_and_one_member_group(blue_noise):
    """Bloom on a two-strip group returns ST_ERR_INVALID (set, and as the last tick took it); the group renders once it is off; a
    one-member group blooms as the single engine does."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA8_SRGB
    w, h = 128, 96
    sc = scenes.cornell(w, h)
    grp = strolle_b200.MultiEngine([0, 0], blue_noise=blue_noise)
    cn = scenes.apply(grp, sc)
    out = np.zeros((h, w, 4), np.uint8)
    grp.set_option(OPT_BLOOM, 1)
    with pytest.raises(Exception, match="BLOOM"):
        grp.render_camera(cn, out, FORMAT_RGBA8_SRGB)
    grp.tick()
    grp.set_option(OPT_BLOOM, 0)
    with pytest.raises(Exception, match="BLOOM"):
        grp.render_camera(cn, out, FORMAT_RGBA8_SRGB)
    grp.tick()
    grp.render_camera(cn, out, FORMAT_RGBA8_SRGB)
    one, solo = strolle_b200.MultiEngine([0], blue_noise=blue_noise), _gpu_engine(blue_noise, exact=False)
    c1, cs = scenes.apply(one, sc), scenes.apply(solo, sc)
    for eng in (one, solo):
        eng.set_option(OPT_BLOOM, 1); eng.set_bloom(intensity=0.4)
    for f in range(3):
        one.tick(); solo.tick()
        a, b = np.zeros((h, w, 4), np.uint8), np.zeros((h, w, 4), np.uint8)
        one.render_camera(c1, a, FORMAT_RGBA8_SRGB); solo.render_camera(cs, b, FORMAT_RGBA8_SRGB)
        assert (a == b).all(), f"frame {f}"
