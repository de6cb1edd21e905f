"""The environment map (st_set_environment_map): the lookup's acos / atan2 against float64, the oracle extension against the oracle and
against the float64 restatement of the lookup at every site that evaluates the sky (tests/ref64_envmap.py), the extension's
deliberate mistakes, known answers, and the CUDA path against the extension (the map as uploaded, ops 8 and 9, every camera buffer of
the strict tier, Reference mode, the product tier, clearing, the instantiation choice together with the other options, row strips)."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle import pyoracle
from oracle_envmap import pyoracle_envmap as E
from tests import ref64_envmap as R
from tests.util import CAMERA_BUFFERS, assert_bits_equal, rel_l2

STAT_ENVIRONMENT_MAP_LAUNCHES = 13
OPT_NORMAL_MAPS, OPT_LIGHT_GRID, OPT_TEXTURE_FILTER = 14, 16, 17


def _scene(name, w, h, rotation=0.0, sun=None, **kw):
    """env_courtyard, or tiled_ground lit by the same sky; `sun` overrides the sun (azimuth, altitude)."""
    sc = getattr(scenes, name)(w, h, **kw)
    sc["environment_map"] = dict(rgba=scenes.courtyard_sky(), intensity=1.5, rotation=rotation)
    if sun is not None:
        sc["sun"] = sun
    return sc


MOVING = {"env_courtyard": 334, "tiled_ground": 313}


def _step(engines, scene, f, w, h):
    """Frame f: the camera moves (env_courtyard: its orbit; tiled_ground: a drift), one instance moves; then tick and render."""
    c = scene["camera"]
    if scene["name"] == "env_courtyard":
        xf, inst_xf = scenes.env_courtyard_motion(f)
    else:
        t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
        t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
        xf, inst_xf = t.reshape(-1), np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.03 * f, 0.0, 0.02 * f], np.float32)
    inst = MOVING[scene["name"]]
    _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == inst)
    for e, cam in engines:
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
        e.insert_instance(inst, mesh, mat, inst_xf)
        e.tick(); e.render_camera(cam)


def _oracle(blue_noise, scene, mutation=None):
    eo = E.EnvMapOracleEngine(blue_noise=blue_noise, mutation=mutation)
    return eo, scenes.apply(eo, scene)


def _probe_run(blue_noise, scene, w, h, frames, mutation=None):
    eo, co = _oracle(blue_noise, scene, mutation)
    eo.probes = []
    for f in range(frames):
        _step([(eo, co)], scene, f, w, h)
    m = scene["environment_map"]
    tex = np.asarray(m["rgba"], np.float32)
    rot = float(np.float32(E.parse(eo.read_environment_map())[3]))
    recs = np.concatenate([r for _, _, r in eo.probes]) if eo.probes else np.zeros((0, E.PROBE_WORDS), np.float32)
    return R.check_records(recs, tex, np.float32(m["intensity"]), rot)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_acos_atan2_within_ulp_bound():
    """The lookup's acos_x and atan2_x (as the oracle evaluates them: ops 8 and 9 on the device) lie within ACOS_ULP and ATAN2_ULP
    float32 ulps of float64, over a sweep of [-1, 1] with +-1, +-0 and their neighbours, and of atan2 over every quadrant, radii
    from 1e-9 to 150, the axes, signed zeros and both sides of the cut (y = +-0 with x < 0)."""
    x = np.concatenate([np.linspace(-1.0, 1.0, 200001), [1.0, -1.0, 0.0, -0.0, 0.5, -0.5, np.nextafter(np.float32(1), np.float32(0)),
                        np.nextafter(np.float32(-1), np.float32(0)), 1e-30, -1e-30]]).astype(np.float32)
    got = E.envm_math(8, x).astype(np.float64)
    want = np.arccos(x.astype(np.float64))
    assert (np.abs(got - want) <= R.ACOS_ULP * R.ulp32(want)).all()
    rng = np.random.RandomState(1)
    ang, rad = rng.uniform(-np.pi, np.pi, 300000), np.exp(rng.uniform(-20.7, 5.0, 300000))
    y, xx = (np.sin(ang) * rad).astype(np.float32), (np.cos(ang) * rad).astype(np.float32)
    sp = np.array([0.0, -0.0, 1.0, -1.0, 1e-30, -1e-30, 3.0, -3.0], np.float32)
    Y, X = np.meshgrid(sp, sp)
    y, xx = np.concatenate([y, Y.ravel()]), np.concatenate([xx, X.ravel()])
    got = E.envm_math(9, y, xx)
    want = np.arctan2(y.astype(np.float64), xx.astype(np.float64))
    assert (np.abs(got.astype(np.float64) - want) <= R.ATAN2_ULP * R.ulp32(want)).all()
    cut = (y == 0) & (xx < 0)
    assert (np.signbit(got[cut]) == np.signbit(y[cut])).all() and (np.abs(got[cut]) == np.float32(np.pi)).all()


def test_without_map_is_the_oracle(blue_noise):
    """With no map set the extension is the plain oracle in every camera buffer (and after a map is set and cleared again)."""
    w, h = 48, 27
    sc = scenes.env_courtyard(w, h)
    del sc["environment_map"]
    eo, co = _oracle(blue_noise, sc)
    ep = pyoracle.OracleEngine(blue_noise=blue_noise)
    cp = scenes.apply(ep, sc)
    for f in range(4):
        if f == 1:
            eo.set_environment_map(scenes.courtyard_sky(), 1.0, 0.0)
            eo.set_environment_map(None)
        _step([(eo, co), (ep, cp)], sc, f, w, h)
        for n in CAMERA_BUFFERS:
            assert_bits_equal(eo.read_buffer(co, n), ep.read_buffer(cp, n), f"frame {f + 1} {n}")


CASES = [("env_courtyard", 0.0, None), ("env_courtyard", 2.5, None), ("tiled_ground", 0.0, None), ("tiled_ground", 2.5, (1.0, -1.2))]


@pytest.mark.parametrize("name,rotation,sun", CASES)
def test_oracle_inside_float64_bound(blue_noise, name, rotation, sun):
    """K10's sky values, K13's radiances (missed bounces and sky draws, and the sky-or-light decision) and K2's colours at paths that
    leave the scene lie inside the float64 bound, over 6 moving frames at 96x54 (Reference mode at depth 2 for K2).  env_courtyard
    has its sun at -1.2 (the sky draw's probability would be 0 without the map)."""
    w, h = 96, 54
    res, bad = _probe_run(blue_noise, _scene(name, w, h, rotation, sun), w, h, 6)
    ref, bad2 = _probe_run(blue_noise, _scene(name, w, h, rotation, sun, mode=scenes.MODE_REFERENCE, ref_depth=2), w, h, 3)
    print(f"{name} rotation {rotation}: {res['records']} + {ref['records']} records, worst {max(res['worst'], ref['worst']):.3g} of the "
          f"bound, {res['undecided'] + ref['undecided']} undecided; per site {res['sites']} {ref['sites']}")
    assert not bad and not bad2, bad + bad2
    assert {"k10", "k13_miss", "k13_sky"} <= set(res["sites"]) and "k2" in ref["sites"]


@pytest.mark.parametrize("mutation", sorted(E.MUTATIONS))
def test_oracle_mutation_leaves_float64_bound(blue_noise, mutation):
    """Each deliberate mistake (v flipped, atan2(d.z, d.x), the rotation's sign, clamping at the seam, no half-texel centre, the
    intensity dropped, the procedural sky's x20 kept, the sky draw still gated by the sun) is caught."""
    w, h = 64, 36
    _, bad = _probe_run(blue_noise, _scene("env_courtyard", w, h, 2.5), w, h, 4, mutation=mutation)
    assert bad, mutation


def _constant_map(c, w=16, h=8):
    m = np.ones((h, w, 4), np.float32)
    m[..., :3] = c
    return m


def test_constant_map_known_answers(blue_noise):
    """A constant map c at intensity I: K10 sky pixels are exactly c I (1/pi) (diffuse) and +0 (specular); Reference mode sky pixels
    accumulate c I per frame."""
    w, h = 48, 27
    c, I = np.array([0.3, 1.7, 4.25], np.float32), np.float32(1.25)
    sc = _scene("env_courtyard", w, h)
    sc["environment_map"] = dict(rgba=_constant_map(c), intensity=float(I), rotation=1.0)
    eo, co = _oracle(blue_noise, sc)
    eo.tick(); eo.render_camera(co)
    sky = eo.read_buffer(co, "prim_triangle_ids").reshape(-1, 4)[:, 0].view(np.uint32) == 0xffffffff
    assert sky.sum() > 100
    diff = eo.read_buffer(co, "di_diff_samples").reshape(-1, 4)[sky, :3]
    spec = eo.read_buffer(co, "di_spec_samples").reshape(-1, 4)[sky, :3]
    want = (c * I) * (np.float32(1.0) / np.float32(math.pi))
    assert_bits_equal(diff, np.broadcast_to(want, diff.shape), "K10 diffuse")
    assert (spec.view(np.uint32) == 0).all()
    ref = _scene("env_courtyard", w, h, mode=scenes.MODE_REFERENCE, ref_depth=1)
    ref["environment_map"] = sc["environment_map"]
    er, cr = _oracle(blue_noise, ref)
    acc = np.zeros(3, np.float32)
    for f in range(3):
        er.tick(); er.render_camera(cr)
        acc = acc + c * I
        sky = er.read_buffer(cr, "prim_triangle_ids").reshape(-1, 4)[:, 0].view(np.uint32) == 0xffffffff
        col = er.read_buffer(cr, "ref_colors").reshape(-1, 4)[sky]
        assert_bits_equal(col[:, :3], np.broadcast_to(acc, (sky.sum(), 3)), f"reference frame {f + 1}")


SIX = {"+Y": (1.0, 0.0, 0.0), "-Y": (0.0, 1.0, 0.0), "-X": (0.0, 0.0, 1.0), "-Z": (1.0, 1.0, 0.0), "+X": (0.0, 1.0, 1.0), "+Z": (1.0, 0.0, 1.0)}


def six_colour_map():
    """8 x 4: row 0 the zenith colour, row 3 the nadir colour; rows 1 and 2 by column pairs {1, 2} -X, {3, 4} -Z, {5, 6} +X, {7, 0} +Z
    (from the rule: u = 0.25 looking down -X, 0.5 down -Z, 0.75 down +X, 1 = 0 down +Z)."""
    m = np.ones((4, 8, 4), np.float32)
    m[0, :, :3] = SIX["+Y"]; m[3, :, :3] = SIX["-Y"]
    for cols, k in (((1, 2), "-X"), ((3, 4), "-Z"), ((5, 6), "+X"), ((7, 0), "+Z")):
        for r in (1, 2):
            for cc in cols:
                m[r, cc, :3] = SIX[k]
    return m


AXES = {"+X": ((1, 0, 0), (0, 1, 0)), "-X": ((-1, 0, 0), (0, 1, 0)), "+Z": ((0, 0, 1), (0, 1, 0)), "-Z": ((0, 0, -1), (0, 1, 0)),
        "+Y": ((0, 1, 0), (0, 0, 1)), "-Y": ((0, -1, 0), (0, 0, 1))}


def orientation_scene(axis, w=33, h=33):
    """A camera at the origin aimed along `axis` with nothing in view (one small quad far behind it), lit by six_colour_map."""
    fwd, up = AXES[axis]
    back = tuple(-5.0 * a for a in fwd)
    quad = np.stack(scenes._quad((back[0] - 0.1, back[1] - 0.1, back[2]), (back[0] + 0.1, back[1] - 0.1, back[2]),
                                 (back[0] + 0.1, back[1] + 0.1, back[2]), (back[0] - 0.1, back[1] + 0.1, back[2]), (0, 0, 1)))
    cam = dict(mode=scenes.MODE_IMAGE, denoise=False, ref_depth=1, w=w, h=h, transform=scenes.look_at_transform((0, 0, 0), fwd, up),
               projection=scenes.perspective_infinite_reverse_rh(math.pi / 4.0, w / h, 0.1))
    return dict(name="orientation", meshes={240: quad}, materials={140: (scenes.material((0.5, 0.5, 0.5, 1.0)), False)},
                instances=[(340, 240, 140, scenes.IDENTITY_AFFINE)], lights=[], sun=(0.0, -1.2), camera=cam,
                environment_map=dict(rgba=six_colour_map(), intensity=1.0, rotation=0.0))


@pytest.mark.parametrize("axis", sorted(AXES))
def test_orientation_six_colour_map(blue_noise, axis):
    """Looking down each axis, the centre pixel's K10 sky value is that axis's colour of six_colour_map, divided by pi (written from
    the rule, not from the oracle)."""
    w = h = 33
    eo, co = _oracle(blue_noise, orientation_scene(axis, w, h))
    eo.tick(); eo.render_camera(co)
    px = eo.read_buffer(co, "di_diff_samples").reshape(h, w, 4)[h // 2, w // 2, :3]
    np.testing.assert_allclose(px * math.pi, SIX[axis], atol=1e-5)


def test_sun_below_horizon_is_dark(blue_noise):
    """The recipe for lighting from the map alone: with the sun below the horizon (altitude -1.2, and -0.05) the sun light's colour
    is 0 (its transmittance through the ground)."""
    for alt in (-1.2, -0.05):
        eo = pyoracle.OracleEngine(blue_noise=blue_noise)
        sc = scenes.env_courtyard(16, 9)
        sc["sun"] = (0.3, alt)
        del sc["environment_map"]
        scenes.apply(eo, sc)
        eo.tick()
        sun = eo.read_scene("lights").reshape(-1, 28)[0]
        assert (sun[4:7] == 0).all(), (alt, sun[4:8])


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu_engine(blue_noise, exact, fused=None, options=None):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    if fused is not None:
        from strolle_b200.engine import OPT_FUSED_PASSES
        e.set_option(OPT_FUSED_PASSES, int(fused))
    for k, v in (options or {}).items():
        e.set_option(k, v)
    return e


@pytest.mark.gpu
def test_read_scene_round_trip(blue_noise):
    """st_read_scene("environment_map") returns the map as set (the rotation reduced into [0, 2 pi)); clearing, setting again and a
    new size work; invalid arguments are refused and leave the previous map in place."""
    from strolle_b200.engine import StrolleError
    e = _gpu_engine(blue_noise, True)
    scenes.apply(e, scenes.env_courtyard(32, 18))
    e.tick()
    W, H, inten, rot, tex = E.parse(e.read_scene("environment_map"))
    sky = scenes.courtyard_sky()
    assert (W, H, inten) == (256, 128, 1.5) and rot == 0.0
    assert_bits_equal(tex, sky, "texels")
    e.set_environment_map(None); e.tick()
    with pytest.raises(StrolleError):
        e.read_scene("environment_map")
    small = np.random.RandomState(3).uniform(0, 4, size=(5, 7, 4)).astype(np.float32)
    e.set_environment_map(small, 0.5, -1.0); e.tick()
    W, H, inten, rot, tex = E.parse(e.read_scene("environment_map"))
    assert (W, H, inten) == (7, 5, 0.5) and rot == np.float32(2.0 * math.pi - 1.0)
    assert_bits_equal(tex, small, "new size")
    bad = small.copy(); bad[2, 3, 1] = -1.0
    nan = small.copy(); nan[0, 0, 0] = np.nan
    for args in ((bad, 1.0, 0.0), (nan, 1.0, 0.0), (small, -1.0, 0.0), (small, float("inf"), 0.0), (small, 1.0, float("nan")),
                 (np.zeros((1, 16385, 4), np.float32), 1.0, 0.0)):
        with pytest.raises(StrolleError):
            e.set_environment_map(*args)
    e.tick()
    assert_bits_equal(E.parse(e.read_scene("environment_map"))[4], small, "after refused calls")


@pytest.mark.gpu
def test_device_acos_atan2_match_oracle(blue_noise):
    """st_device_math ops 8 and 9 are the oracle's acos_x and atan2_x bit for bit."""
    e = _gpu_engine(blue_noise, True)
    rng = np.random.RandomState(2)
    x = np.concatenate([rng.uniform(-1, 1, 200000), [1, -1, 0, -0.0, 0.5, -0.5]]).astype(np.float32)
    assert_bits_equal(e.device_math("acos_env", x), E.envm_math(8, x), "acos")
    y, xx = rng.normal(size=200000).astype(np.float32), rng.normal(size=200000).astype(np.float32)
    y[:8], xx[:8] = [0, -0.0, 0, -0.0, 1, -1, 0, 0], [-1, -1, 1, 1, 0, 0, -0.0, 0]
    assert_bits_equal(e.device_math("atan2_env", y, xx), E.envm_math(9, y, xx), "atan2")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["env_courtyard", "tiled_ground"])
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
def test_strict_tier_bit_exact_with_oracle(oracle, blue_noise, name, size):
    """A map set, strict arithmetic, 13 frames with the camera and an instance moving, the unfused and fused schedules: every camera
    buffer is the extension's, bit for bit (the fused schedule: every buffer it still writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = size
    scene = _scene(name, w, h, 2.5)
    gs = [_gpu_engine(blue_noise, True, fused=fused) for fused in (False, True)]
    cams = [scenes.apply(g, scene) for g in gs]
    eo, co = _oracle(blue_noise, scene)
    for f in range(13):
        _step([(g, c) for g, c in zip(gs, cams)] + [(eo, co)], scene, f, w, h)
        for fused, g, c in zip((False, True), gs, cams):
            for n in CAMERA_BUFFERS:
                if fused and n in NOT_WRITTEN_WHEN_FUSED:
                    continue
                assert_bits_equal(g.read_buffer(c, n), eo.read_buffer(co, n), f"{name} fused={fused} {size} frame {f + 1} {n}")
    assert all(g.get_stat(STAT_ENVIRONMENT_MAP_LAUNCHES) > 0 for g in gs)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2])
def test_reference_mode_bit_exact_with_oracle(oracle, blue_noise, depth):
    """Reference mode with a map: every camera buffer is the extension's, bit for bit, over 13 moving frames."""
    w, h = 224, 126
    scene = _scene("env_courtyard", w, h, 2.5, mode=scenes.MODE_REFERENCE, ref_depth=depth)
    eg = _gpu_engine(blue_noise, True)
    cg = scenes.apply(eg, scene)
    eo, co = _oracle(blue_noise, scene)
    for f in range(13):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for n in CAMERA_BUFFERS:
            assert_bits_equal(eg.read_buffer(cg, n), eo.read_buffer(co, n), f"depth {depth} frame {f + 1} {n}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["env_courtyard", "tiled_ground"])
def test_product_tier_within_tolerance_of_oracle(oracle, blue_noise, name):
    """A map set, product defaults: the G-buffer is the strict tier's bit for bit, and the composed frame stays within 1e-3 relative
    per-channel L2 of the extension over 13 frames, or, where the frame without a map already drifts further from the oracle than
    that, within 1.5 times that drift."""
    w, h = 224, 126
    worst = {}
    for with_map in (True, False):
        scene = _scene(name, w, h, 2.5)
        if not with_map:
            del scene["environment_map"]
        prod, strict = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, True)
        cp, cs = scenes.apply(prod, scene), scenes.apply(strict, scene)
        eo, co = _oracle(blue_noise, scene)
        worst[with_map] = 0.0
        for f in range(13):
            _step([(prod, cp), (strict, cs), (eo, co)], scene, f, w, h)
            for n in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "prim_triangle_ids"):
                assert_bits_equal(prod.read_buffer(cp, n), strict.read_buffer(cs, n), f"frame {f + 1} {n}")
            a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
            b = eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
            for ch in range(3):
                worst[with_map] = max(worst[with_map], rel_l2(a[:, ch], b[:, ch]))
    print(f"{name}: worst relative L2 with the map {worst[True]:.3g}, without {worst[False]:.3g}")
    assert worst[True] <= max(1e-3, 1.5 * worst[False])


@pytest.mark.gpu
def test_clear_restores_the_procedural_sky(blue_noise):
    """After the map is cleared, from the next tick on, the frame is computed as by an engine that never had one: in Reference mode
    with the camera moving (no state carried between frames) every camera buffer is bit-identical; in the image mode, where the
    ReSTIR reservoirs and the denoiser's history still carry radiance gathered under the map until they are replaced, K10's sky
    pixels are; a map set and cleared before any tick leaves every buffer as it was; nothing counts as a map launch any more."""
    w, h = 96, 54
    for mode in (scenes.MODE_REFERENCE, scenes.MODE_IMAGE):
        scene = _scene("env_courtyard", w, h, 1.0, mode=mode, ref_depth=2)
        plain = dict(scene); del plain["environment_map"]
        a, b = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, False)
        ca, cb = scenes.apply(a, scene), scenes.apply(b, plain)
        for f in range(6):
            if f == 3:
                a.set_environment_map(None)
            _step([(a, ca), (b, cb)], scene, f, w, h)
            if f < 3:
                continue
            if mode == scenes.MODE_REFERENCE:
                for n in CAMERA_BUFFERS:
                    assert_bits_equal(a.read_buffer(ca, n), b.read_buffer(cb, n), f"reference frame {f + 1} {n}")
            else:
                sky = b.read_buffer(cb, "prim_triangle_ids").reshape(-1, 4)[:, 0].view(np.uint32) == 0xffffffff
                assert sky.sum() > 100
                for n in ("di_diff_samples", "di_spec_samples"):
                    assert_bits_equal(a.read_buffer(ca, n).reshape(-1, 4)[sky], b.read_buffer(cb, n).reshape(-1, 4)[sky], f"frame {f + 1} {n}")
        launches = a.get_stat(STAT_ENVIRONMENT_MAP_LAUNCHES)
        _step([(a, ca)], scene, 6, w, h)
        assert launches > 0 and a.get_stat(STAT_ENVIRONMENT_MAP_LAUNCHES) == launches
    scene = _scene("env_courtyard", w, h, 1.0)
    plain = dict(scene); del plain["environment_map"]
    a, b = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, False)
    ca, cb = scenes.apply(a, scene), scenes.apply(b, plain)
    a.set_environment_map(None)
    for f in range(3):
        _step([(a, ca), (b, cb)], scene, f, w, h)
        for n in CAMERA_BUFFERS:
            assert_bits_equal(a.read_buffer(ca, n), b.read_buffer(cb, n), f"cleared before the first tick, frame {f + 1} {n}")
    assert a.get_stat(STAT_ENVIRONMENT_MAP_LAUNCHES) == 0


@pytest.mark.gpu
def test_with_other_options(blue_noise):
    """Normal maps, texture filtering and the light grid on together with the map: K10's sky pixels are the map-only run's, bit for
    bit (the ENVM instantiation composes with NMAP, TEXF and LGRID)."""
    w, h = 224, 126
    sc = _scene("tiled_ground", w, h, 2.5)
    sc["images"] = dict(sc["images"]); sc["images"][725] = scenes.brick_normal_map()
    sc["material_textures"] = {k: dict(v) for k, v in sc["material_textures"].items()}
    sc["material_textures"][111]["normal_map"] = 725
    both = _gpu_engine(blue_noise, True, options={OPT_NORMAL_MAPS: 1, OPT_TEXTURE_FILTER: 1, OPT_LIGHT_GRID: 8})
    only = _gpu_engine(blue_noise, True)
    cb, co = scenes.apply(both, sc), scenes.apply(only, sc)
    for f in range(3):
        _step([(both, cb), (only, co)], sc, f, w, h)
        sky = only.read_buffer(co, "prim_triangle_ids").reshape(-1, 4)[:, 0].view(np.uint32) == 0xffffffff
        assert sky.sum() > 1000
        for n in ("di_diff_samples", "di_spec_samples"):
            assert_bits_equal(both.read_buffer(cb, n).reshape(-1, 4)[sky], only.read_buffer(co, n).reshape(-1, 4)[sky], f"frame {f + 1} {n}")
    assert both.get_stat(8) > 0   # the NMAP instantiations ran


def _devices(n):
    import torch
    have = max(torch.cuda.device_count(), 1)
    return [k % have for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,size", [(2, (320, 288)), (3, (256, 400))])
def test_row_strips_match_single_gpu(blue_noise, n, size):
    """A map set, env_courtyard as n row strips (st_multi_*, devices reused when there are fewer), camera and crate moving: every
    camera buffer is the single-GPU frame's, bit for bit, over 7 frames."""
    import strolle_b200
    w, h = size
    scene = _scene("env_courtyard", w, h, 2.5)
    one = _gpu_engine(blue_noise, False)
    grp = strolle_b200.MultiEngine(_devices(n), blue_noise=blue_noise)
    c1, cn = scenes.apply(one, scene), scenes.apply(grp, scene)
    for f in range(7):
        _step([(one, c1), (grp, cn)], scene, f, w, h)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(cn, name), one.read_buffer(c1, name), f"{n} strips frame {f + 1} {name}")
    assert grp.peer_errors(cn) == 0
