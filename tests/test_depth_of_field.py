"""Depth of field (ST_OPT_DEPTH_OF_FIELD, st_set_depth_of_field): the oracle extension against known answers written from the rule and
against the float64 restatement (with its deliberate mistakes); the CUDA path against the extension (strict tier bit for bit, product
tier within the option-off drift), its refusals, lifetime and isolation, and the strip entry points."""
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
from oracle_dof import pyoracle_dof as D
from tests import ref64_dof as RD

OPT_TONEMAPPING, OPT_AUTO_EXPOSURE, OPT_BLOOM, OPT_DEPTH_OF_FIELD, STAT_GATHERS = 20, 21, 22, 23, 17
OPT_FUSED_PASSES, OPT_TEMPORAL_AA = 11, 18
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SH = 0.01866


def _u32(words):
    return np.asarray(words, np.float32).view(np.uint32)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_constants_agree_across_header_python_and_rust():
    from strolle_b200 import engine as E
    header = open(os.path.join(ROOT, "include", "strolle_b200.h")).read()
    rust = open(os.path.join(ROOT, "rust", "strolle-b200-sys", "src", "lib.rs")).read()
    for name, value in (("OPT_DEPTH_OF_FIELD", 23), ("STAT_DEPTH_OF_FIELD_GATHERS", 17)):
        assert re.search(rf"ST_{name} = {value}\b", header), name
        assert f"pub const ST_{name}: c_int = {value};" in rust, name
        assert getattr(E, name) == value and getattr(D, name) == value
    assert "pub fn st_set_depth_of_field(e: *mut st_engine, dof: *const st_depth_of_field) -> c_int;" in rust
    assert "pub fn st_multi_set_depth_of_field(m: *mut st_multi, dof: *const st_depth_of_field) -> c_int;" in rust
    assert "pub struct st_depth_of_field" in rust
    assert list(E.DEPTH_OF_FIELD_DEFAULTS) == list(D.FIELDS) and E.DEPTH_OF_FIELD_DEFAULTS == D.DEFAULTS
    assert re.search(r"NULL restores the defaults \{10, 1, 0\.01866, 16\}", header)
    hl = open(os.path.join(ROOT, "rust", "strolle-b200", "src", "lib.rs")).read()
    assert "pub fn set_depth_of_field(&mut self, dof: Option<&DepthOfField>)" in hl and "pub struct DepthOfField" in hl
    bevy = open(os.path.join(ROOT, "rust", "bevy-strolle-b200", "src", "lib.rs")).read()
    assert "pub depth_of_field: Option<st::DepthOfField>" in bevy


def test_tap_table_restated():
    """The extension's tap table is the float64 restatement's: the centre, then rings of 8 j taps at rho j / 4, rounded offsets."""
    dxy, d = D.taps()
    rdxy, rd = RD.taps()
    assert (dxy == rdxy).all() and (d.view(np.uint32) == rd.view(np.uint32)).all()
    assert (dxy[:, 0] == 0).all() and (np.abs(dxy).max(axis=(1, 2)) == np.arange(1, 33)).all()
    assert (np.abs(D.taps("offsets_truncated")[0] - dxy).sum() > 0)


# A synthetic frame: a pinhole camera at the origin looking down -Z, and a hit distance per pixel
def _camera(w, h, fov_y=math.radians(50.0)):
    return scenes.look_at_transform((0.0, 0.0, 0.0), (0.0, 0.0, -1.0)), scenes.perspective_infinite_reverse_rh(fov_y, w / h, 0.1)


def _synthetic(w, h, depth_of_px, colour_of_px):
    """(output, t, camera40, transform, projection): a view depth z per pixel turned into hit distances along the pixel's ray."""
    xf, pr = _camera(w, h)
    c40 = _gpu_camera(xf, pr, w, h)
    d = D.rays(c40, w, h).astype(np.float64)
    fw = np.array([0.0, 0.0, -1.0])
    z = depth_of_px.astype(np.float64)
    t = np.where(z > 0, z / (d @ fw), 0.0).astype(np.float32)
    out = np.zeros((h, w, 4), np.float32)
    out[..., :3] = colour_of_px
    out[..., 3] = 1.0
    return out, t, c40, xf, pr


def _gpu_camera(xf, pr, w, h):
    """GpuCamera (40 floats) of a transform and projection, as the oracle serialises it."""
    eo = pyoracle.OracleEngine(blue_noise=scenes.blue_noise())
    cam = eo.create_camera(0, True, 1, w, h, xf, pr)
    return eo.read_buffer(cam, "curr_camera")


def _lens_for(pr, h, F, k, R=16.0):
    """Settings with focal distance F whose k (the CoC at infinity before the clamp) is k pixels."""
    f = 0.5 * SH * float(np.float32(pr[5]))
    N = f * f / (F - f) * h / SH / 2.0 / k
    return D.params(focal_distance=F, aperture_f_stops=N, sensor_height=SH, max_radius=R)


def _check(out, t, c40, xf, pr, p, w, h, mutation=None):
    words, frame = D.run(out, t, c40, w, h, p, xf, pr, mutation)
    bad, undecided = RD.check(words, frame, out, t, D.rays(c40, w, h), p, xf, pr, h, w)
    return words, frame, bad, undecided


def test_constant_frame_stays_constant():
    """A constant frame at any depths stays constant within the float64 bound."""
    w, h = 70, 45
    z = (2.0 + 30.0 * np.random.RandomState(3).rand(h, w)).astype(np.float32)
    z[5:20, 10:30] = 0.0   # sky
    c = np.array([0.3, 0.7, 1.9], np.float32)
    out, t, c40, xf, pr = _synthetic(w, h, z, c)
    p = _lens_for(pr, h, 6.0, 20.0, R=12.0)
    words, frame, bad, undecided = _check(out, t, c40, xf, pr, p, w, h)
    assert bad == 0 and undecided == 0
    assert np.allclose(frame[..., :3], c, rtol=200 * 2.0 ** -24, atol=0)
    assert (D.run(out, t, c40, w, h, p, xf, pr)[1] == frame).all()


def test_wall_on_the_focus_plane_is_copied():
    """A wall on the focus plane: every |r| < 1/2, every rho 0, and the frame is `output` bit for bit; so is F <= f."""
    w, h = 50, 37
    out, t, c40, xf, pr = _synthetic(w, h, np.full((h, w), 5.0, np.float32), np.float32(0))
    out[..., :3] = np.random.RandomState(4).rand(h, w, 3).astype(np.float32) * 4
    p = _lens_for(pr, h, 5.0, 50.0)
    words, frame, bad, _ = _check(out, t, c40, xf, pr, p, w, h)
    parsed = _parse(words)
    assert bad == 0 and np.abs(parsed["r"]).max() < 0.5 and (parsed["rho"] == 0).all() and parsed["defocused"]
    assert (frame.view(np.uint32) == out.view(np.uint32)).all()
    f = 0.5 * SH * float(pr[5])
    p2 = D.params(focal_distance=float(np.float32(f * 0.9)), aperture_f_stops=0.01, sensor_height=SH)
    words, frame = D.run(out, t, c40, w, h, p2, xf, pr)
    parsed = _parse(words)
    assert not parsed["defocused"] and parsed["k"] == 0 and (parsed["r"] == 0).all() and (frame.view(np.uint32) == out.view(np.uint32)).all()


def _parse(words):
    from strolle_b200.engine import parse_depth_of_field
    return parse_depth_of_field(words)


def test_lone_bright_pixel_spreads_into_a_disc():
    """A lone bright pixel on a far plane spreads over a disc of radius about r (to the pixels whose 81 taps reach it), with its energy
    conserved within 15 % (the gather normalises per receiving pixel, not per emitter)."""
    w, h = 96, 96
    z = np.full((h, w), 40.0, np.float32)
    out, t, c40, xf, pr = _synthetic(w, h, z, np.float32(0))
    out[48, 48, :3] = 1000.0
    p = _lens_for(pr, h, 4.0, 8.0)
    words, frame, bad, undecided = _check(out, t, c40, xf, pr, p, w, h)
    assert bad == 0 and undecided == 0
    r = float(_parse(words)["r"][48, 48])
    assert 6.0 < r < 8.0
    e = frame[..., 0].astype(np.float64)
    assert abs(e.sum() / 1000.0 - 1.0) < 0.15, e.sum()
    yy, xx = np.mgrid[0:h, 0:w]
    dist = np.hypot(yy - 48, xx - 48)
    lit = dist[e > 0]
    assert e[dist > r + 1.5].sum() == 0 and lit.max() >= r - 1.5 and lit.size >= 32   # the taps that see it, across the whole disc


def test_in_focus_foreground_keeps_its_colour():
    """An in-focus foreground half over a blurred background: every foreground pixel keeps its colour within the float64 bound (no
    background colour), while the background blurs across its own half."""
    w, h = 80, 48
    z = np.full((h, w), 60.0, np.float32)
    z[:, :40] = 5.0
    col = np.zeros((h, w, 3), np.float32)
    col[:, :40] = (0.0, 1.0, 0.0)
    col[:, 40:] = (1.0, 0.0, 0.0)
    col[::3, 40:] = (0.0, 0.0, 4.0)
    out, t, c40, xf, pr = _synthetic(w, h, z, col)
    p = _lens_for(pr, h, float(np.float32(5.0)), 10.0, R=10.0)
    words, frame, bad, undecided = _check(out, t, c40, xf, pr, p, w, h)
    assert bad == 0 and undecided == 0
    r = _parse(words)["r"]
    fg = np.abs(r[:, :40]) < 0.05
    assert fg.all()
    assert np.abs(frame[:, :40, 0]).max() < 1e-5 and np.abs(frame[:, :40, 2]).max() < 1e-5
    assert np.ptp(frame[10:38, 50:70, 2]) < 0.5 * np.ptp(out[10:38, 50:70, 2])


def test_blurred_near_object_spreads_over_the_background():
    """A blurred near square spreads over the in-focus background behind it by about its radius."""
    w, h = 96, 64
    z = np.full((h, w), 20.0, np.float32)
    z[24:40, 40:56] = 1.0
    col = np.zeros((h, w, 3), np.float32)
    col[24:40, 40:56] = 1.0
    out, t, c40, xf, pr = _synthetic(w, h, z, col)
    p = _lens_for(pr, h, float(np.float32(20.0)), 8.0, R=6.0)
    words, frame, bad, undecided = _check(out, t, c40, xf, pr, p, w, h)
    assert bad == 0 and undecided == 0
    r = _parse(words)["r"]
    assert (r[24:40, 40:56] == -6.0).all()
    row = frame[32, :, 0]
    spread = np.flatnonzero(row > 0.01)
    assert 40 - 7 <= spread.min() <= 40 - 3 and 55 + 3 <= spread.max() <= 55 + 7, spread


def test_nan_and_inf_taps_read_zero():
    """NaN and inf channels of neighbouring taps read 0: the same gathered bits as 0 there, outside the pixel itself."""
    w, h = 40, 40
    z = (3.0 + 20 * np.random.RandomState(9).rand(h, w)).astype(np.float32)
    out, t, c40, xf, pr = _synthetic(w, h, z, np.float32(0.5))
    p = _lens_for(pr, h, 6.0, 12.0, R=8.0)
    bad = out.copy()
    bad[10, 10, :3] = np.nan
    bad[20, 25, 1] = np.inf
    zero = out.copy()
    zero[10, 10, :3] = 0.0
    zero[20, 25, 1] = 0.0
    fb, fz = D.run(bad, t, c40, w, h, p, xf, pr)[1], D.run(zero, t, c40, w, h, p, xf, pr)[1]
    assert (fb.view(np.uint32) == fz.view(np.uint32)).all()
    assert np.isnan(D.run(bad, t, c40, w, h, p, xf, pr, "nan_kept")[1]).any()


def _ref_lens(sc, spread=0.02):
    """Reference mode's lens for a scene: focus at the camera's distance to the origin, an aperture radius of `spread` times it."""
    c = sc["camera"]
    F = float(np.float32(np.linalg.norm(np.asarray(c["transform"], np.float64)[12:15])))
    f = 0.5 * SH * float(np.float32(c["projection"][5]))
    return D.params(focal_distance=F, aperture_f_stops=f / (2.0 * spread * F), sensor_height=SH)


def test_reference_lens_ray_against_float64():
    """Reference mode's thin-lens rays: every origin lies inside the aperture disc (radius A / 2 on the right and up axes, none along
    the view axis) and every ray passes through the pinhole ray's point at view depth F, within a float64 bound; the draws cover the disc."""
    w, h = 64, 40
    xf, pr = _camera(w, h)
    xf = scenes.look_at_transform((0.3, 0.2, 1.0), (0.0, 0.0, -4.0))
    c40 = _gpu_camera(xf, pr, w, h)
    p = D.params(focal_distance=4.0, aperture_f_stops=0.05, sensor_height=SH)
    on, L = D.lens(p, xf, pr)
    assert on
    hA, F = float(L[0]), float(L[1])
    right, up, fwd = (L[2 + 3 * k:5 + 3 * k].astype(np.float64) for k in range(3))
    pin_o, _ = D.lens_rays(c40, w, h, np.concatenate([[0.0], L[1:]]).astype(np.float32), 0)   # h = 0: the pinhole origins, exactly
    d = D.rays(c40, w, h).astype(np.float64)
    o, dirs = (a.astype(np.float64) for a in D.lens_rays(c40, w, h, L, D.dispatch_seed(0xC0FFEE, 5, D.LENS_DISPATCH)))
    U = 2.0 ** -24
    off = o - pin_o.astype(np.float64)
    a, b, z = off @ right, off @ up, off @ fwd
    scale = 8 * U * (np.abs(pin_o).sum(-1) + hA)
    assert (np.hypot(a, b) <= hA * (1 + 8 * U) + scale).all() and (np.abs(z) <= scale).all()
    assert np.hypot(a, b).max() > 0.9 * hA and (a > 0.5 * hA).any() and (a < -0.5 * hA).any() and (b > 0.5 * hA).any() and (b < -0.5 * hA).any()
    pf = pin_o + d * (F / (d @ fwd))[..., None]
    v = pf - o
    t = (v * dirs).sum(-1)
    miss = np.linalg.norm(v - dirs * t[..., None], axis=-1)
    bound = 16 * U * (np.linalg.norm(v, axis=-1) + np.abs(pf).sum(-1) + np.abs(o).sum(-1))
    assert (miss <= bound).all(), float((miss / bound).max())
    assert (np.abs(np.linalg.norm(dirs, axis=-1) - 1.0) <= 4 * U).all()


def test_reference_lens_stream(blue_noise):
    """Reference mode with the lens accumulates a different image from the pinhole's, and drawing the lens from the shading stream (a
    deliberate mistake) changes it again; F <= f renders through the pinhole."""
    w, h = 40, 30
    sc = scenes.cornell(w, h, mode=scenes.MODE_REFERENCE)
    frames = {}
    for key, opt, mutation, p in (("pin", 0, None, None), ("lens", 1, None, _ref_lens(sc, 0.05)), ("shading", 1, "lens_shading_stream", _ref_lens(sc, 0.05)),
                                  ("inside", 1, None, D.params(focal_distance=1e-3, aperture_f_stops=0.05, sensor_height=SH))):
        x = D.DofOracle(pyoracle.OracleEngine(blue_noise=blue_noise), mutation)
        x.set_option(OPT_DEPTH_OF_FIELD, opt)
        if p:
            x.set_depth_of_field(**p)
        cam = scenes.apply(x, sc)
        for _ in range(2):
            x.tick(); x.render_camera(cam)
        frames[key] = x.frame(cam).copy()
    assert (frames["inside"].view(np.uint32) == frames["pin"].view(np.uint32)).all()
    assert (frames["lens"] != frames["pin"]).any() and (frames["shading"] != frames["lens"]).any()


SCENES = {"cornell": scenes.cornell, "dungeon": scenes.dungeon, "env_sunlit": scenes.env_sunlit, "aa_edges": scenes.aa_edges}


def _moving(sc, f):
    t = np.asarray(sc["camera"]["transform"], np.float32).reshape(4, 4).copy()
    t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
    return t.reshape(-1)


def _scene_frames(name, blue_noise, w=48, h=27, frames=13):
    """The oracle's (output, t, camera, transform, projection) over 13 moving frames."""
    sc = SCENES[name](w, h)
    eo = EM.EnvMapOracleEngine(blue_noise=blue_noise) if "environment_map" in sc else pyoracle.OracleEngine(blue_noise=blue_noise)
    x = D.DofOracle(eo)
    cam = scenes.apply(x, sc)
    c = sc["camera"]
    outs = []
    for f in range(frames):
        xf = _moving(sc, f)
        x.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
        x.tick(); x.render_camera(cam)
        outs.append((x.read_buffer(cam, "output").reshape(h, w, 4).copy(), x.depth(cam).copy(), x.read_buffer(cam, "curr_camera").copy(), xf,
                     np.asarray(c["projection"], np.float32)))
    return outs


def _case_lens(frames, R):
    """A focus in the middle of the scene's depths and a k of 2 R: near and far both blur, some to the clamp."""
    out, t, c40, xf, pr = frames[0]
    h = out.shape[0]
    hit = t[t > 0]
    F = float(np.float32(np.median(hit))) if hit.size else 5.0
    return _lens_for(pr, h, F, 2.0 * R, R=R)


@pytest.fixture(scope="module")
def scene_frames(blue_noise):
    frames = {n: _scene_frames(n, blue_noise) for n in SCENES}
    frames["odd"] = _scene_frames("cornell", blue_noise, w=37, h=23, frames=4)
    return frames


def _violations(frames, R, mutation=None):
    bad = und = n = 0
    p = _case_lens(frames, R)
    for out, t, c40, xf, pr in frames:
        h, w = out.shape[:2]
        b, u = _check(out, t, c40, xf, pr, p, w, h, mutation)[2:]
        bad += b; und += u; n += w * h
    return bad, und / n


@pytest.mark.parametrize("name", list(SCENES) + ["odd"])
def test_extension_inside_the_float64_bound(scene_frames, name):
    """On cornell, dungeon, env_sunlit and aa_edges over 13 moving frames (and an odd 37x23 size), for max_radius 1, 16 and 32, the
    extension's words and frame lie inside the float64 bound; at most 5 % of the pixels are undecided."""
    for R in (1.0, 16.0, 32.0):
        bad, undecided = _violations(scene_frames[name], R)
        assert bad == 0 and undecided <= 0.05, (name, R, bad, undecided)


@pytest.mark.parametrize("mutation", ["coc_sign", "ray_distance", "no_background_limit", "no_density", "no_dilation", "offsets_truncated",
                                      "sky_in_focus"])
def test_deliberate_mistakes_leave_the_bound(scene_frames, mutation):
    """Each deliberate mistake, run through the same frames, leaves the float64 bound somewhere."""
    assert sum(_violations(scene_frames[n][:4], R, mutation)[0] for n in ("env_sunlit", "dungeon", "cornell") for R in (8.0, 32.0)) > 0


def test_nan_kept_leaves_the_bound(scene_frames):
    out, t, c40, xf, pr = scene_frames["env_sunlit"][0]
    out = out.copy()
    h, w = out.shape[:2]
    p = _case_lens(scene_frames["env_sunlit"], 16.0)
    rho = _parse(D.run(out, t, c40, w, h, p, xf, pr)[0])["rho"]
    ty, tx = np.argwhere(rho > 0)[0]
    out[ty * 16 + 3, tx * 16 + 3, 1] = np.nan
    assert _check(out, t, c40, xf, pr, p, w, h, "nan_kept")[2] > 0
    assert _check(out, t, c40, xf, pr, p, w, h)[2] == 0


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


def _rgba32(e, cam, w, h):
    from strolle_b200.engine import FORMAT_RGBA32F
    out = np.zeros((h, w, 4), np.float32)
    e.copy_output(cam, out, FORMAT_RGBA32F)
    return out


def _gpu_lens(e, cam, sc, R):
    w, h = sc["camera"]["w"], sc["camera"]["h"]
    t = e.read_buffer(cam, "surface_nd").reshape(h, w, 4)[..., 3]
    return t, _lens_for(np.asarray(sc["camera"]["projection"], np.float32), h,
                        float(np.float32(np.median(t[t > 0]))) if (t > 0).any() else 5.0, 2.0 * R, R=R)


def _run_pair(blue_noise, sc, R, frames=13, fused=False, op=0, auto=False, bloom=False, taa=False, exact=True):
    """The device and the extension (over the device's own `output`, `surface_nd` and camera) over `frames` moving frames: the
    "depth_of_field" words, the Rgba32F frame and the Rgba8 frame, bit for bit."""
    w, h = sc["camera"]["w"], sc["camera"]["h"]
    opts = {OPT_TONEMAPPING: op, OPT_AUTO_EXPOSURE: int(auto), OPT_TEMPORAL_AA: int(taa), OPT_BLOOM: int(bloom), OPT_DEPTH_OF_FIELD: 1}
    e = _gpu_engine(blue_noise, exact=exact, fused=fused, opts=opts)
    x = B.BloomOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    for k in (OPT_TONEMAPPING, OPT_AUTO_EXPOSURE, OPT_BLOOM):
        x.set_option(k, opts[k])
    c = sc["camera"]
    cg = scenes.apply(e, sc)
    cx = x.create_camera(c["mode"], c["denoise"], c["ref_depth"], w, h, c["transform"], c["projection"])
    p = None
    for f in range(frames):
        xf = _moving(sc, f)
        e.update_camera(cg, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
        e.tick(); x.tick()
        e.render_camera(cg)
        if p is None:
            p = _gpu_lens(e, cg, sc, R)[1]
            e.set_depth_of_field(**p)   # from the next frame on; this one defocuses with the defaults
        lens = p if f > 0 else D.params()
        t = e.read_buffer(cg, "surface_nd").reshape(h, w, 4)[..., 3]
        words, frame = D.run(e.read_buffer(cg, "output"), t, e.read_buffer(cg, "curr_camera"), w, h, lens, xf, c["projection"])
        gw = _u32(e.read_buffer(cg, "depth_of_field"))
        assert gw.size == words.size and (gw == _u32(words)).all(), f"frame {f}: {int((gw != _u32(words)).sum())} words differ"
        got = _rgba32(e, cg, w, h)
        assert (got.view(np.uint32) == frame.view(np.uint32)).all(), f"frame {f}: {int((got != frame).any(-1).sum())} pixels differ"
        if x.x.meters(cx):
            x.x.meter_output(cx, frame)
        if bloom:
            x.build_pyramid(cx, frame)
        g8, w8 = _rgba8(e, cg, w, h), x.rgba8(cx, frame)
        assert (g8 == w8).all(), f"frame {f}: {int((g8 != w8).any(-1).sum())} Rgba8 pixels differ"
    return e, cg


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1.0, 16.0, 32.0])
def test_gpu_strict_bit_exact(blue_noise, R):
    """Strict tier: the words, the Rgba32F frame and the Rgba8 bytes equal the extension's over 13 moving frames at 224x126 (unfused)
    and 67x45 (fused, with tonemapping and auto exposure)."""
    _run_pair(blue_noise, scenes.cornell(224, 126), R)
    _run_pair(blue_noise, scenes.env_sunlit(67, 45), R, fused=True, op=4, auto=True)


@pytest.mark.gpu
def test_gpu_strict_bloom_taa_and_scenes(blue_noise):
    """With bloom, with temporal AA (the jittered camera's rays), and on dungeon and aa_edges at an odd size."""
    _run_pair(blue_noise, scenes.env_sunlit(96, 54), 16.0, frames=5, op=3, auto=True, bloom=True)
    _run_pair(blue_noise, scenes.cornell(96, 64), 8.0, frames=5, taa=True, op=2)
    _run_pair(blue_noise, scenes.dungeon(37, 23), 32.0, frames=4)
    _run_pair(blue_noise, scenes.aa_edges(96, 64), 4.0, frames=4)


@pytest.mark.gpu
def test_gpu_product_tier(blue_noise):
    """Product tier (the default fast-math kernels): the G-buffer stays bit-exact; the Rgba32F frame stays within max(1e-3, 1.5 x the
    option-off drift) relative per-channel L2 of the extension run end to end on the oracle; the CoC and gather kernels are exact on the
    product frame's own `output` and `surface_nd`."""
    from tests.util import rel_l2
    w, h = 160, 90
    sc = scenes.env_sunlit(w, h)
    e = _gpu_engine(blue_noise, exact=False, opts={OPT_DEPTH_OF_FIELD: 1})
    x = D.DofOracle(EM.EnvMapOracleEngine(blue_noise=blue_noise))
    x.set_option(OPT_DEPTH_OF_FIELD, 1)
    cg, cx = scenes.apply(e, sc), scenes.apply(x, sc)
    c = sc["camera"]
    p = None
    for f in range(9):
        xf = _moving(sc, f)
        for eng, cam in ((e, cg), (x, cx)):
            eng.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
            eng.tick()
        e.render_camera(cg); x.render_camera(cx)
        for name in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b"):
            assert (e.read_buffer(cg, name).view(np.uint32) == x.base.read_buffer(cx, name).view(np.uint32)).all(), f"frame {f}: {name}"
        lens = p or D.params()
        t = e.read_buffer(cg, "surface_nd").reshape(h, w, 4)[..., 3]
        assert (t.view(np.uint32) == x.depth(cx).view(np.uint32)).all()
        dev_out = e.read_buffer(cg, "output")
        words, frame = D.run(dev_out, t, e.read_buffer(cg, "curr_camera"), w, h, lens, xf, c["projection"])
        assert (_u32(e.read_buffer(cg, "depth_of_field")) == _u32(words)).all(), f"frame {f}: words on the product frame"
        got = _rgba32(e, cg, w, h)
        assert (got.view(np.uint32) == frame.view(np.uint32)).all(), f"frame {f}: gather on the product frame"
        want, ora_out = x.frame(cx), x.read_buffer(cx, "output").reshape(h, w, 4)
        for ch in range(3):
            drift, err = rel_l2(dev_out.reshape(h, w, 4)[..., ch], ora_out[..., ch]), rel_l2(got[..., ch], want[..., ch])
            assert err <= max(1e-3, 1.5 * drift), f"frame {f} channel {ch}: {err:.2e} against option-off drift {drift:.2e}"
        if p is None:
            p = _gpu_lens(e, cg, sc, 16.0)[1]
            e.set_depth_of_field(**p); x.set_depth_of_field(**p)


@pytest.mark.gpu
def test_gpu_strict_reference_lens(blue_noise):
    """Strict tier, Reference mode with the lens: the accumulated frame and ref_colors equal the extension's bit for bit over 5 still
    frames (ref_depth 1 and 2), and the lens drawn from the shading stream (a deliberate mistake) does not."""
    for depth, (w, h) in ((1, (64, 48)), (2, (37, 23))):
        sc = scenes.cornell(w, h, mode=scenes.MODE_REFERENCE, ref_depth=depth)
        p = _ref_lens(sc, 0.04)
        e = _gpu_engine(blue_noise, opts={OPT_DEPTH_OF_FIELD: 1})
        x = D.DofOracle(pyoracle.OracleEngine(blue_noise=blue_noise))
        bad = D.DofOracle(pyoracle.OracleEngine(blue_noise=blue_noise), "lens_shading_stream")
        for eng in (x, bad):
            eng.set_option(OPT_DEPTH_OF_FIELD, 1)
        cg, cx, cb = scenes.apply(e, sc), scenes.apply(x, sc), scenes.apply(bad, sc)
        for eng in (e, x, bad):
            eng.set_depth_of_field(**p)
        for f in range(5):
            for eng, cam in ((e, cg), (x, cx), (bad, cb)):
                eng.tick(); eng.render_camera(cam)
            got = _rgba32(e, cg, w, h)
            assert (got.view(np.uint32) == x.frame(cx).view(np.uint32)).all(), f"depth {depth} frame {f}: {int((got != x.frame(cx)).any(-1).sum())} pixels"
            assert (e.read_buffer(cg, "ref_colors").view(np.uint32) == x.base.read_buffer(cx, "ref_colors").view(np.uint32)).all()
            assert (got != bad.frame(cb)).any()
        assert e.read_buffer(cg, "ref_colors").reshape(h, w, 4)[..., 3].min() == 5.0   # accumulated while the camera is still


INVALID = (dict(focal_distance=math.nan), dict(aperture_f_stops=math.inf), dict(sensor_height=-math.inf), dict(max_radius=math.nan),
           dict(focal_distance=0.0), dict(focal_distance=-1.0), dict(aperture_f_stops=0.0), dict(sensor_height=-0.01), dict(max_radius=0.5),
           dict(max_radius=32.5), dict(max_radius=-4.0))


@pytest.mark.gpu
def test_gpu_refusals_change_nothing(blue_noise):
    """Option values outside 0..1 and every out-of-range field are refused, on an engine and on a group; an engine that received every
    refused call renders the same frame and words as one that never did."""
    import strolle_b200
    for bad in (-1, 2):
        with pytest.raises(strolle_b200.StrolleError):
            _gpu_engine(blue_noise).set_option(OPT_DEPTH_OF_FIELD, bad)
    w, h = 96, 54
    sc = scenes.cornell(w, h)
    a, b = _gpu_engine(blue_noise, opts={OPT_DEPTH_OF_FIELD: 1}), _gpu_engine(blue_noise, opts={OPT_DEPTH_OF_FIELD: 1})
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    for e in (a, b):
        e.set_depth_of_field(focal_distance=3.0, aperture_f_stops=0.02, max_radius=12.0)
    for f in range(3):
        for fields in INVALID:
            with pytest.raises(strolle_b200.StrolleError, match="st_set_depth_of_field"):
                a.set_depth_of_field(**fields)
        with pytest.raises(strolle_b200.StrolleError):
            a.set_option(OPT_DEPTH_OF_FIELD, 3)
        a.tick(); b.tick(); a.render_camera(ca); b.render_camera(cb)
        assert (_rgba32(a, ca, w, h).view(np.uint32) == _rgba32(b, cb, w, h).view(np.uint32)).all(), f"frame {f}"
        assert (_u32(a.read_buffer(ca, "depth_of_field")) == _u32(b.read_buffer(cb, "depth_of_field"))).all(), f"frame {f}"
    grp = strolle_b200.MultiEngine([0, 0], blue_noise=blue_noise)
    for fields in INVALID:
        with pytest.raises(strolle_b200.StrolleError, match="st_set_depth_of_field"):
            grp.set_depth_of_field(**fields)
    grp.set_depth_of_field(max_radius=32.0)
    grp.set_depth_of_field()


@pytest.mark.gpu
def test_gpu_option_off_lifetime_heatmap_isolation_and_statistic(blue_noise):
    """`output` never changes with the option on; turning it off stores today's frame again and frees the buffer; one gather per
    rendered frame and none per copy; the buffer restarts zeroed after a resize; two cameras do not interfere; the heat map is not
    defocused; Reference mode samples the lens (its frame changes) and has no gathered frame."""
    import strolle_b200
    w, h = 96, 54
    sc = scenes.cornell(w, h)
    a, b = _gpu_engine(blue_noise), _gpu_engine(blue_noise, opts={OPT_DEPTH_OF_FIELD: 1})
    ca, cb = scenes.apply(a, sc), scenes.apply(b, sc)
    k = sc["camera"]
    b.set_depth_of_field(focal_distance=3.0, aperture_f_stops=0.02, max_radius=12.0)
    c2 = b.create_camera(k["mode"], k["denoise"], k["ref_depth"], 61, 37, k["transform"], k["projection"])
    for f in range(5):
        if f == 3:
            b.set_option(OPT_DEPTH_OF_FIELD, 0)
        a.tick(); b.tick()
        if f == 0:
            with pytest.raises(strolle_b200.StrolleError):
                b.read_buffer(cb, "depth_of_field")   # allocated by the first render or copy
            assert (_rgba32(b, cb, w, h) == 0).all()   # zero-filled
        a.render_camera(ca); b.render_camera(cb)
        assert (a.read_buffer(ca, "output").view(np.uint32) == b.read_buffer(cb, "output").view(np.uint32)).all()
        same = (_rgba32(a, ca, w, h).view(np.uint32) == _rgba32(b, cb, w, h).view(np.uint32)).all()
        assert same == (f >= 3), f"frame {f}"
        if f == 1:
            b.render_camera(c2)
            n = b.get_stat(STAT_GATHERS)
            first = _u32(b.read_buffer(cb, "depth_of_field")).copy()
            _rgba32(b, cb, w, h); _rgba8(b, cb, w, h)
            assert n == 3 and b.get_stat(STAT_GATHERS) == n   # copies never gather
            words2 = _u32(b.read_buffer(c2, "depth_of_field"))
            assert words2[0] == 61 and words2[1] == 37 and (_u32(b.read_buffer(cb, "depth_of_field")) == first).all()
    assert b.get_stat(STAT_GATHERS) == 4   # frames 0, 1 (and the second camera once), 2
    with pytest.raises(strolle_b200.StrolleError):
        b.read_buffer(cb, "depth_of_field")
    b.set_option(OPT_DEPTH_OF_FIELD, 1)
    b.update_camera(cb, k["mode"], k["denoise"], k["ref_depth"], w + 2, h, k["transform"], k["projection"])
    a.tick(); b.tick()   # the engines stay on the same frame: Reference mode's draws follow it
    assert (_rgba32(b, cb, w + 2, h) == 0).all()   # reallocated zeroed at the new size
    b.render_camera(cb)
    assert _u32(b.read_buffer(cb, "depth_of_field"))[0] == w + 2
    hm = [eng.create_camera(scenes.MODE_BVH_HEATMAP, False, 1, w, h, k["transform"], k["projection"]) for eng in (a, b)]
    a.tick(); b.tick()
    a.render_camera(hm[0]); b.render_camera(hm[1])
    assert (_rgba32(a, hm[0], w, h).view(np.uint32) == _rgba32(b, hm[1], w, h).view(np.uint32)).all()
    assert (_rgba8(a, hm[0], w, h) == _rgba8(b, hm[1], w, h)).all()
    with pytest.raises(strolle_b200.StrolleError):
        b.read_buffer(hm[1], "depth_of_field")
    rf = [eng.create_camera(scenes.MODE_REFERENCE, False, 1, w, h, k["transform"], k["projection"]) for eng in (a, b)]
    a.tick(); b.tick()
    a.render_camera(rf[0]); b.render_camera(rf[1])
    assert (_rgba32(a, rf[0], w, h) != _rgba32(b, rf[1], w, h)).any()   # Reference mode samples the lens: no gather, no buffer
    with pytest.raises(strolle_b200.StrolleError):
        b.read_buffer(rf[1], "depth_of_field")


@pytest.mark.gpu
@pytest.mark.parametrize("members", [2, 3])
def test_gpu_strips_refused_and_one_member_group(blue_noise, members):
    """The option on a strip group returns ST_ERR_INVALID (set, and as the last tick took it); the group renders once it is off; a
    one-member group defocuses as the single engine does."""
    import strolle_b200
    from strolle_b200.engine import FORMAT_RGBA32F
    w, h = 128, 96
    sc = scenes.cornell(w, h)
    grp = strolle_b200.MultiEngine([0] * members, blue_noise=blue_noise)
    cn = scenes.apply(grp, sc)
    out = np.zeros((h, w, 4), np.float32)
    grp.set_option(OPT_DEPTH_OF_FIELD, 1)
    with pytest.raises(Exception, match="DEPTH_OF_FIELD"):
        grp.render_camera(cn, out, FORMAT_RGBA32F)
    grp.tick()
    grp.set_option(OPT_DEPTH_OF_FIELD, 0)
    with pytest.raises(Exception, match="DEPTH_OF_FIELD"):
        grp.render_camera(cn, out, FORMAT_RGBA32F)
    grp.tick()
    grp.render_camera(cn, out, FORMAT_RGBA32F)
    one, solo = strolle_b200.MultiEngine([0], blue_noise=blue_noise), _gpu_engine(blue_noise, exact=False)
    c1, cs = scenes.apply(one, sc), scenes.apply(solo, sc)
    for eng in (one, solo):
        eng.set_option(OPT_DEPTH_OF_FIELD, 1); eng.set_depth_of_field(focal_distance=3.0, aperture_f_stops=0.02)
    for f in range(3):
        one.tick(); solo.tick()
        a, b = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 4), np.float32)
        one.render_camera(c1, a, FORMAT_RGBA32F); solo.render_camera(cs, b, FORMAT_RGBA32F)
        assert (a.view(np.uint32) == b.view(np.uint32)).all(), f"frame {f}"
