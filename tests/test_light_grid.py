"""Light grid (ST_OPT_LIGHT_GRID): the oracle's grid (oracle_lightgrid/) against a float64 restatement of the rule, the zero
radiance of every dropped light, unbiasedness, the option off; on the GPU the device grid against the oracle's word for word, the
strict tier bit for bit, the product tier, Cornell unchanged, noise, and row strips."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle_lightgrid import pyoracle_lightgrid as P
from tests.util import CAMERA_BUFFERS, assert_bits_equal, rel_l2

OPT_LIGHT_GRID, STAT_LIGHT_GRID_BUILDS = 16, 10
BIG, TINY = 2.0 ** 60, 2.0 ** -60


# ---- float64 restatement ----------------------------------------------------------------------------------------------------------

def _lights(e):
    """(slots, light_count) of what the engine's frames see: slots = n x 28 float32."""
    lc = int(e.read_scene("world").view(np.uint32)[0])
    return e.read_scene("lights").reshape(-1, 28), lc


def _cullable(L):
    kind = L[:, 8].view(np.uint32)
    with np.errstate(invalid="ignore"):
        return ((kind == 1) & (np.abs(L[:, 0:3]) <= BIG).all(1) & np.isfinite(L[:, 4:7]).all(1) & (L[:, 7] >= TINY) & (L[:, 7] <= BIG))


def _check_grid(words, L, lc, n):
    """The rule, restated: header (f32, the host's operations), then every list checked in float64."""
    g = P.parse(words)
    L = L[:lc]
    cull = _cullable(L)
    assert g["light_count"] == lc and g["K"] == P.K
    f32 = np.float32
    if not cull.any():
        assert g["dims"] == (0, 0, 0) and g["cells"] == 0
    else:
        c, r = L[cull, 0:3], L[cull, 7:8]
        lo, hi = (c - r).min(0), (c + r).max(0)
        ext = (hi - lo).astype(f32)
        longest = ext.max()
        m = max(np.abs(lo).max(), np.abs(hi).max())
        ulp = np.spacing(f32(m))
        dims = np.clip(np.ceil((f32(n) * ext) / longest), 1, n).astype(np.uint32)
        assert tuple(int(d) for d in dims) == g["dims"]
        cell = (ext / dims.astype(f32)).astype(f32)
        assert_bits_equal(g["lo"], lo, "lo"); assert_bits_equal(g["cell"], cell, "cell")
        assert_bits_equal(g["inv_cell"], (dims.astype(f32) / ext).astype(f32), "inv_cell")
        assert_bits_equal(g["margin"], (cell * f32(0.015625) + f32(8.0) * ulp).astype(f32), "margin")
        assert_bits_equal(g["band"], (f32(0.0078125) + (f32(2.0) * ulp) * g["inv_cell"]).astype(f32), "band")
    non = np.flatnonzero(~cull)
    counts, lists = g["counts"], g["lists"]
    # the outside list: the non-cullable slots, or overflow
    if len(non) > P.K:
        assert counts[-1] == P.OVERFLOW
    else:
        assert counts[-1] == len(non) and (lists[-1][:len(non)] == non).all() and (lists[-1][len(non):] == P.OVERFLOW).all()
    if g["cells"] == 0:
        return g
    D = np.array(g["dims"])
    lo64, cell64 = g["lo"].astype(np.float64), g["cell"].astype(np.float64)
    ulp64 = float(np.spacing(np.float32(max(np.abs(g["lo"]).max(), np.abs(g["lo"] + g["cell"] * D).max()))))
    slack = cell64 * (1.0 / 128 + 2.0 ** -15) + 4.0 * ulp64     # how far outside its cell a point the lookup maps there can lie
    idx = np.stack(np.meshgrid(np.arange(D[0]), np.arange(D[1]), np.arange(D[2]), indexing="ij"), -1).reshape(-1, 3)
    cid = (idx[:, 2] * D[1] + idx[:, 1]) * D[0] + idx[:, 0]
    bmin, bmax = lo64 + idx * cell64, lo64 + (idx + 1) * cell64
    cs = np.flatnonzero(cull)
    C64, R64 = L[cs, 0:3].astype(np.float64), L[cs, 7].astype(np.float64)
    checked = 0
    for k in range(len(cid)):
        cnt, lst = counts[cid[k]], lists[cid[k]]
        d_exact = np.linalg.norm(np.maximum(np.maximum(bmin[k] - C64, C64 - bmax[k]), 0.0), axis=1)
        d_slack = np.linalg.norm(np.maximum(np.maximum((bmin[k] - slack) - C64, C64 - (bmax[k] + slack)), 0.0), axis=1)
        if cnt == P.OVERFLOW:   # more than K slots the rule could keep (cell grown by the margin, range by 2^-7)
            mg = g["margin"].astype(np.float64) * 1.001
            d_grown = np.linalg.norm(np.maximum(np.maximum((bmin[k] - mg) - C64, C64 - (bmax[k] + mg)), 0.0), axis=1)
            assert len(non) + int((d_grown <= R64 * (1.0 + 2.0 ** -7)).sum()) > P.K
            continue
        ids = lst[:cnt]
        assert (lst[cnt:] == P.OVERFLOW).all()
        assert (np.diff(ids.astype(np.int64)) > 0).all(), "ascending"
        assert np.isin(non, ids).all(), "every non-cullable slot"
        inc = np.isin(cs, ids)
        # every dropped light is out of reach of every point the cell hands out, with room to spare for f32 and the fast build
        assert (d_slack[~inc] ** 2 > R64[~inc] ** 2 * (1.0 + 2.0 ** -10)).all(), f"cell {cid[k]}: a dropped light reaches the cell"
        # every kept light comes within its range plus the cell diagonal
        assert (d_exact[inc] <= R64[inc] + np.linalg.norm(cell64)).all(), f"cell {cid[k]}: a kept light is far out of reach"
        checked += 1
    assert checked + int((counts[:-1] == P.OVERFLOW).sum()) == len(cid)
    return g


def _grid_oracle(blue_noise, scene, n, mutation=None):
    eo = P.LightGridOracleEngine(blue_noise=blue_noise, mutation=mutation)
    cam = scenes.apply(eo, scene)
    eo.set_light_grid(n)
    return eo, cam


def _huge_range(scene):
    s = dict(scene); s["lights"] = list(scene["lights"]) + [(999, scenes.LIGHT_POINT, scenes.point_light((0.0, 1.0, 0.0), 0.2, (5.0, 5.0, 5.0), 1.0e4))]
    return s


def _only_infinite(scene):
    s = dict(scene)
    s["lights"] = [(h, k, np.concatenate([p[:7], [np.inf], p[8:]]).astype(np.float32)) for h, k, p in scene["lights"]]
    return s


def _rounding_scene():
    """Three lights on the x axis: the box is [-11, 11] x [-1, 1]^2 (cells of 1 at N = 22), the middle light's sphere ends 2^-23 short
    of the cell face x = 1 and the right light's sphere touches the box face x = 11, so points a few ulp inside those spheres map to
    the next cell (or outside) unless the margins are right.  The sun stands high."""
    mat = {100: (scenes.material((0.8, 0.8, 0.8, 1.0)), False)}
    lights = [(400, scenes.LIGHT_POINT, scenes.point_light((-10.0, 0.0, 0.0), 0.1, (3.0, 3.0, 3.0), 1.0)),
              (401, scenes.LIGHT_POINT, scenes.point_light((0.0, 0.0, 0.0), 0.1, (3.0, 3.0, 3.0), 1.0 - 2.0 ** -23)),
              (402, scenes.LIGHT_POINT, scenes.point_light((10.0, 0.0, 0.0), 0.1, (3.0, 3.0, 3.0), 1.0))]
    cam = dict(mode=scenes.MODE_IMAGE, denoise=True, ref_depth=1, w=32, h=32, transform=scenes.look_at_transform((0.0, 3.0, 12.0), (0.0, 0.0, 0.0)),
               projection=scenes.perspective_infinite_reverse_rh(math.pi / 4.0, 1.0, 0.1))
    return dict(name="rounding", meshes={200: np.stack(scenes._box((-12.0, -3.0, -2.0), (12.0, -2.0, 2.0)))}, materials=mat,
                instances=[(300, 200, 100, scenes.IDENTITY_AFFINE)], lights=lights, sun=(0.5, 0.8), camera=cam)


GRID_SCENES = {
    "stress_lights": lambda: scenes.stress_lights(32, 32, t=0.7),
    "demo_level": lambda: scenes.demo_level(32, 32),
    "cornell_spots": lambda: scenes.cornell_spots(32, 32),
    "huge_range": lambda: _huge_range(scenes.stress_lights(32, 32)),
    "only_infinite": lambda: _only_infinite(scenes.cornell(32, 32)),
    "rounding": _rounding_scene,
}


# ---- CPU ----------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(GRID_SCENES))
@pytest.mark.parametrize("n", [1, 7, 32, 64])
def test_oracle_grid_matches_float64_rule(blue_noise, name, n):
    """The oracle's grid: its header is the rule's f32 arithmetic; every list is ascending, holds every non-cullable slot, drops only
    lights that are out of reach in float64 of every point the lookup can map to the cell, keeps only lights within range plus the
    cell diagonal; overflow and the outside list are right."""
    eo, _ = _grid_oracle(blue_noise, GRID_SCENES[name](), n)
    eo.tick()
    L, lc = _lights(eo)
    g = _check_grid(eo.read_light_grid(), L, lc, n)
    if name == "huge_range" and n >= 7:
        assert (g["counts"][:-1] == P.OVERFLOW).any()
    if name == "only_infinite":
        assert g["cells"] == 0
    if name == "stress_lights" and n == 32:
        c = g["counts"][:-1]
        assert (c != P.OVERFLOW).all() and c.max() < 16 and c.min() >= 1


def _probe_points(g, rng, n_random=4000):
    """Grid vertices and cell-face centres nudged by -4..4 ulp per axis, and random points around the box."""
    D = np.array(g["dims"]); lo, cell = g["lo"], g["cell"]
    ax = [lo[a] + cell[a] * np.arange(0, D[a] + 1, 0.5, dtype=np.float32) for a in range(3)]
    base = np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    if len(base) > 3000:
        base = base[rng.choice(len(base), 3000, replace=False)]
    pts = [base]
    for k in (-4, -1, 1, 4):
        for a in range(3):
            p = base.copy()
            p[:, a] = np.nextafter(p[:, a], np.float32(np.inf) if k > 0 else np.float32(-np.inf))
            for _ in range(abs(k) - 1):
                p[:, a] = np.nextafter(p[:, a], np.float32(np.inf) if k > 0 else np.float32(-np.inf))
            pts.append(p)
    hi = lo + cell * D
    pad = 0.1 * (hi - lo)
    pts.append(rng.uniform(lo - pad, hi + pad, size=(n_random, 3)).astype(np.float32))
    return np.concatenate(pts)


def _sphere_extremes(L, lc):
    """Each cullable light's six axis extremes pulled 1..4 ulp inside its sphere."""
    cull = np.flatnonzero(_cullable(L[:lc]))
    pts = []
    for i in cull:
        c, r = L[i, 0:3], L[i, 7]
        for a in range(3):
            for s in (-1.0, 1.0):
                p = c.copy(); p[a] = np.float32(c[a] + s * r)
                for k in range(4):
                    p = p.copy(); p[a] = np.nextafter(p[a], c[a]); pts.append(p)
    return np.array(pts, np.float32).reshape(-1, 3)


def _hit_points(eo, scene, rng, n=3000):
    """Closest hits of camera rays through the frame."""
    c = scene["camera"]
    eye = np.asarray(c["transform"], np.float32).reshape(4, 4)[3, :3]
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((n, 8), np.float32); rays[:, 0:3] = eye; rays[:, 4:7] = d; rays[:, 3] = np.float32(3.4028234663852886e38)
    h = eo.trace_closest(rays).reshape(n, 12)
    ok = np.isfinite(h[:, 8]) & (h[:, 8] < 1e30)
    return (rays[ok, 0:3] + rays[ok, 4:7] * h[ok, 8:9]).astype(np.float32)


def _zero_check(eo, scene, rng):
    """For every probe point and every slot missing from its list, the oracle's light_radiance (shading normal towards the light) is
    exactly +-0.  Returns the number of (point, light) pairs that were checked and of those that were not zero."""
    L, lc = _lights(eo)
    g = P.parse(eo.read_light_grid())
    parts = [_sphere_extremes(L, lc), _hit_points(eo, scene, rng)]
    if g["cells"]:
        parts.append(_probe_points(g, rng))
    pts = np.concatenate(parts)
    n, ids = eo.point_lists(pts)
    P_, I_ = [], []
    for s in range(lc):
        missing = (n != P.OVERFLOW) & ~(ids == s).any(1)
        P_.append(np.flatnonzero(missing)); I_.append(np.full(missing.sum(), s, np.uint32))
    pi, li = np.concatenate(P_), np.concatenate(I_)
    p = pts[pi]
    to = L[li, 0:3].astype(np.float32) - p
    nrm = (to / np.maximum(np.linalg.norm(to, axis=1, keepdims=True), 1e-30)).astype(np.float32)
    rad = eo.radiance(p, nrm, li)
    return len(pi), int((rad != 0).any(1).sum())


@pytest.mark.parametrize("name", ["stress_lights", "demo_level", "cornell_spots", "rounding"])
def test_dropped_lights_have_zero_radiance(blue_noise, name):
    """Every light missing from a point's list has exactly zero radiance there: grid vertices and face centres nudged by 1-4 ulp,
    sphere extremes pulled inside, random points and camera-ray hits."""
    scene = GRID_SCENES[name]()
    rng = np.random.RandomState(5)
    for n in (7, 22, 64):
        eo, _ = _grid_oracle(blue_noise, scene, n)
        eo.tick()
        checked, nonzero = _zero_check(eo, scene, rng)
        assert checked > 1000 and nonzero == 0, (n, checked, nonzero)


@pytest.mark.parametrize("mutation,name,n", [("no_margin", "rounding", 22), ("no_band", "rounding", 22), ("drop_sun", "demo_level", 32)])
def test_zero_check_catches_mistakes(blue_noise, mutation, name, n):
    """Each deliberate mistake - cells not grown by the margin (and no range slack), the point -> cell index without its band, the
    sun left out of the lists - gives some dropped light a nonzero radiance at a probe point."""
    scene = GRID_SCENES[name]()
    eo, _ = _grid_oracle(blue_noise, scene, n, mutation=mutation)
    eo.tick()
    _, nonzero = _zero_check(eo, scene, np.random.RandomState(5))
    assert nonzero > 0


def _tile_stats(frames, tile=8):
    f = np.asarray(frames, np.float64)            # frames x h x w
    F, h, w = f.shape
    return f[:, :h // tile * tile, :w // tile * tile].reshape(F, h // tile, tile, w // tile, tile).mean((2, 4)).reshape(F, -1)


def _unbiased(on, off, z=5.0):
    """Paired per-tile batch means: |mean(on - off)| within z batch standard errors (plus a tiny floor) in every tile."""
    d = on - off
    se = d.std(0, ddof=1) / math.sqrt(len(d))
    return np.abs(d.mean(0)) <= z * se + 1e-6 * np.abs(off.mean(0)) + 1e-9


def _ref_frames(e, cam, w, h, frames):
    """Per-frame Reference-mode estimates (luma of this frame's path radiance), read from the accumulation."""
    out, prev = [], np.zeros((h, w))
    for _ in range(frames):
        e.tick(); e.render_camera(cam)
        acc = e.read_buffer(cam, "ref_colors").reshape(h, w, 4)[..., :3].astype(np.float64).sum(-1)
        out.append(acc - prev); prev = acc
    return np.array(out)


@pytest.mark.parametrize("mutation", [None, "global_pdf"])
def test_oracle_reference_mode_unbiased(blue_noise, mutation):
    """Reference mode, stress_lights at 48x48, depth 1, static lights: per 8x8 tile, the option-on batch mean agrees with the
    option-off one within 5 batch standard errors; K2 with pdf = 1 / light_count over the grid's list fails the same test."""
    w = h = 48
    scene = scenes.stress_lights(w, h, mode=scenes.MODE_REFERENCE, ref_depth=1, t=0.3)
    on, con = _grid_oracle(blue_noise, scene, 32, mutation=mutation)
    off, coff = _grid_oracle(blue_noise, scene, 0)
    a, b = _ref_frames(on, con, w, h, 96), _ref_frames(off, coff, w, h, 96)
    ok = _unbiased(_tile_stats(a), _tile_stats(b))
    assert b.mean() > 0
    if mutation is None:
        assert ok.all(), np.flatnonzero(~ok)
    else:
        assert not ok.all()


def test_oracle_option_off_is_the_oracle(oracle, blue_noise):
    """With the option off, oracle_lightgrid's buffers are the plain oracle's, bit for bit, over 4 frames of stress_lights."""
    scene = scenes.stress_lights(40, 32)
    a = P.LightGridOracleEngine(blue_noise=blue_noise)
    b = oracle.OracleEngine(blue_noise=blue_noise)
    ca, cb = scenes.apply(a, scene), scenes.apply(b, scene)
    for f in range(4):
        for e, c in ((a, ca), (b, cb)):
            e.tick(); e.render_camera(c)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(a.read_buffer(ca, name), b.read_buffer(cb, name), f"frame {f + 1} {name}")


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------

def _gpu(blue_noise, exact, n=32, fused=None):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    e.set_option(OPT_LIGHT_GRID, n)
    if fused is not None:
        from strolle_b200.engine import OPT_FUSED_PASSES
        e.set_option(OPT_FUSED_PASSES, int(fused))
    return e


def _move_lights(engines, t):
    for e in engines:
        for h, kind, params in scenes.stress_lights_lights(t):
            e.insert_light(h, kind, params)


@pytest.mark.gpu
def test_option_values(blue_noise):
    """0..64 are accepted, anything else is ST_ERR_INVALID; no grid can be read while the option is off."""
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise)
    for v in (0, 1, 64):
        e.set_option(OPT_LIGHT_GRID, v)
    for v in (-1, 65, 1000):
        with pytest.raises(strolle_b200.StrolleError):
            e.set_option(OPT_LIGHT_GRID, v)
    e.set_option(OPT_LIGHT_GRID, 0)
    scenes.apply(e, scenes.cornell(32, 32)); e.tick()
    with pytest.raises(strolle_b200.StrolleError):
        e.read_scene("light_grid")


@pytest.mark.gpu
def test_device_grid_equals_oracle(blue_noise):
    """After every tick - lights moved and recoloured, inserted, removed, the sun changed, spot lights added, N changed - the device
    grid (st_read_scene) is the oracle's word for word; a tick that changes neither lights nor N builds nothing."""
    scene = scenes.stress_lights(32, 32)
    eg, eo = _gpu(blue_noise, True), P.LightGridOracleEngine(blue_noise=blue_noise)
    scenes.apply(eg, scene); scenes.apply(eo, scene); eo.set_light_grid(32)

    def check(what, n=32):
        eg.tick(); eo.tick()
        a, b = eg.read_scene("light_grid").view(np.uint32), eo.read_light_grid()
        assert a.shape == b.shape and (a == b).all(), f"{what}: {int((a != b).sum()) if a.shape == b.shape else (a.shape, b.shape)} words differ"
        L, lc = _lights(eo)
        _check_grid(b, L, lc, n)

    check("first tick")
    check("second tick (the light mirror uploads once more after an insert)")
    builds = eg.get_stat(STAT_LIGHT_GRID_BUILDS)
    eg.tick(); eo.tick()
    assert eg.get_stat(STAT_LIGHT_GRID_BUILDS) == builds, "nothing changed: no build"
    for t in (0.4, 1.3):
        _move_lights((eg, eo), t); check(f"moved t={t}")
    for e in (eg, eo):
        e.insert_light(900, scenes.LIGHT_POINT, scenes.point_light((30.0, 140.0, 5.0), 0.3, (9.0, 1.0, 1.0), 35.0))
        e.insert_light(901, scenes.LIGHT_SPOT, scenes.spot_light((-20.0, 60.0, 10.0), 0.2, (3.0, 3.0, 9.0), 25.0, (0.0, -1.0, 0.0), 0.6))
    check("inserted a point and a spot light")
    for e in (eg, eo):
        e.remove_light(410); e.remove_light(455)
    check("removed two")
    for e in (eg, eo):
        e.update_sun(0.3, 0.7)
    check("sun changed")
    for e in (eg, eo):
        e.remove_light(900)
    eg.set_option(OPT_LIGHT_GRID, 7); eo.set_light_grid(7)
    check("N = 7", 7)


def _step(engines, f, moving=True):
    if moving:
        _move_lights([e for e, _ in engines], 0.5 + 0.05 * f)
    for e, cam in engines:
        e.tick(); e.render_camera(cam)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True])
def test_strict_tier_bit_exact_with_oracle(oracle, blue_noise, fused):
    """Option on, strict arithmetic, stress_lights at 96x64 with the lights moving and recolouring, 13 frames: every camera buffer is
    oracle_lightgrid's bit for bit (the fused schedule: every buffer it writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = 96, 64
    scene = scenes.stress_lights(w, h, t=0.5)
    eg = _gpu(blue_noise, True, fused=fused)
    eo, co = _grid_oracle(blue_noise, scene, 32)
    cg = scenes.apply(eg, scene)
    names = [n for n in CAMERA_BUFFERS if not (fused and n in NOT_WRITTEN_WHEN_FUSED)]
    for f in range(13):
        _step([(eg, cg), (eo, co)], f)
        for name in names:
            assert_bits_equal(eg.read_buffer(cg, name), eo.read_buffer(co, name), f"fused={fused} frame {f + 1} {name}")
    assert eg.get_stat(STAT_LIGHT_GRID_BUILDS) == 13


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2])
def test_reference_mode_bit_exact_with_oracle(oracle, blue_noise, depth):
    """Reference mode with the option on, lights moving: rays, hits and accumulated colours are the oracle's, bit for bit."""
    w, h = 96, 64
    scene = scenes.stress_lights(w, h, mode=scenes.MODE_REFERENCE, ref_depth=depth, t=0.5)
    eg = _gpu(blue_noise, True)
    eo, co = _grid_oracle(blue_noise, scene, 32)
    cg = scenes.apply(eg, scene)
    for f in range(6):
        _step([(eg, cg), (eo, co)], f)
        for name in ("ref_hits", "ref_rays", "ref_colors", "output"):
            assert_bits_equal(eg.read_buffer(cg, name), eo.read_buffer(co, name), f"depth {depth} frame {f + 1} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["stress_lights", "demo_level"])
def test_product_tier_within_tolerance_of_oracle(oracle, blue_noise, name):
    """Option on, product defaults, 13 frames: the G-buffer is the strict tier's bit for bit and the composed frame stays within 1e-3
    relative per-channel L2 of oracle_lightgrid."""
    w, h = 128, 72
    scene = scenes.stress_lights(w, h, t=0.5) if name == "stress_lights" else scenes.demo_level(w, h)
    prod, strict = _gpu(blue_noise, False), _gpu(blue_noise, True)
    cp, cs = scenes.apply(prod, scene), scenes.apply(strict, scene)
    eo, co = _grid_oracle(blue_noise, scene, 32)
    worst = 0.0
    for f in range(13):
        for e, cam in ((prod, cp), (strict, cs), (eo, co)):
            e.tick(); e.render_camera(cam)
        for b in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "surface_nd", "prim_triangle_ids"):
            assert_bits_equal(prod.read_buffer(cp, b), strict.read_buffer(cs, b), f"frame {f + 1} {b}")
        a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
        o = eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
        for ch in range(3):
            worst = max(worst, rel_l2(a[:, ch], o[:, ch]))
    print(f"{name}: worst per-channel relative L2 {worst:.3g}")
    assert worst <= 1e-3


@pytest.mark.gpu
def test_cornell_unchanged(blue_noise):
    """Cornell: its light reaches every hit, so every list a hit looks up is [0, 1], the identity - option on and off are
    bit-identical in every camera buffer, Image and Reference mode, strict and product tier."""
    for exact in (True, False):
        for mode in (scenes.MODE_IMAGE, scenes.MODE_REFERENCE):
            scene = scenes.cornell(96, 64, mode=mode)
            on, off = _gpu(blue_noise, exact), _gpu(blue_noise, exact, n=0)
            con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
            for f in range(5):
                on.tick(); off.tick(); on.render_camera(con); off.render_camera(coff)
                for name in CAMERA_BUFFERS:
                    assert_bits_equal(on.read_buffer(con, name), off.read_buffer(coff, name), f"exact={exact} mode={mode} frame {f + 1} {name}")
            g = P.parse(on.read_scene("light_grid").view(np.uint32))
            D = np.array(g["dims"])
            centre = ((np.array([0.0, 1.5, 0.5]) - g["lo"]) * g["inv_cell"]).astype(int)   # the light's own cell, and every cell near it
            near = [(z * D[1] + y) * D[0] + x for z in range(centre[2] - 3, centre[2] + 4) for y in range(centre[1] - 3, centre[1] + 4)
                    for x in range(centre[0] - 3, centre[0] + 4)]
            assert (g["counts"][near] == 2).all() and (g["lists"][near, :2] == [0, 1]).all()
            assert (g["lists"][:-1, 0] == 0).all(), "the sun is in every list"


@pytest.mark.gpu
def test_reference_mode_unbiased_and_less_noisy(blue_noise):
    """Reference mode, stress_lights at 128x128, depth 1, static lights, 128 frames: per 8x8 tile the option-on batch mean agrees
    with the option-off one within 5 batch standard errors, and the per-frame variance is lower with the option on."""
    w = h = 128
    scene = scenes.stress_lights(w, h, mode=scenes.MODE_REFERENCE, ref_depth=1, t=0.3)
    on, off = _gpu(blue_noise, False), _gpu(blue_noise, False, n=0)
    con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
    a, b = _ref_frames(on, con, w, h, 128), _ref_frames(off, coff, w, h, 128)
    ok = _unbiased(_tile_stats(a), _tile_stats(b))
    assert ok.all(), np.flatnonzero(~ok)
    var_on, var_off = a.var(0).mean(), b.var(0).mean()
    print(f"reference-mode per-pixel variance: on {var_on:.4g} off {var_off:.4g} ratio {var_on / var_off:.4g}")
    assert var_on < var_off


@pytest.mark.gpu
def test_restir_di_noise_lower(blue_noise):
    """MODE_DI_DIFFUSE without denoising, static lights: one frame's relative L2 against the 256-frame mean is lower with the option on."""
    w, h = 128, 128
    scene = scenes.stress_lights(w, h, mode=scenes.MODE_DI_DIFFUSE, denoise=False, t=0.3)
    res = {}
    for n in (32, 0):
        e = _gpu(blue_noise, False, n=n)
        cam = scenes.apply(e, scene)
        frames = []
        for _ in range(256):
            e.tick(); e.render_camera(cam)
            frames.append(e.read_buffer(cam, "output").reshape(h, w, 4)[..., :3].astype(np.float64))
        mean = np.mean(frames, 0)
        res[n] = float(np.mean([rel_l2(frames[k], mean) for k in (63, 127, 191)]))
    print(f"ReSTIR DI single-frame relative L2 vs the 256-frame mean: on {res[32]:.4g} off {res[0]:.4g}")
    assert res[32] < res[0]


def _devices(n):
    import torch
    have = max(torch.cuda.device_count(), 1)
    return [k % have for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,size", [(2, (320, 288)), (3, (256, 400))])
def test_row_strips_match_single_gpu(blue_noise, n, size):
    """Option on, stress_lights as n row strips (st_multi_*, devices reused when there are fewer), lights moving: every camera
    buffer is the single-GPU frame's, bit for bit, over 7 frames."""
    import strolle_b200
    w, h = size
    scene = scenes.stress_lights(w, h, t=0.5)
    one = _gpu(blue_noise, False)
    grp = strolle_b200.MultiEngine(_devices(n), blue_noise=blue_noise)
    grp.set_option(OPT_LIGHT_GRID, 32)
    c1, cn = scenes.apply(one, scene), scenes.apply(grp, scene)
    for f in range(7):
        _move_lights((one, grp), 0.5 + 0.05 * f)
        for e, cam in ((one, c1), (grp, cn)):
            e.tick(); e.render_camera(cam)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(cn, name), one.read_buffer(c1, name), f"{n} strips frame {f + 1} {name}")
    assert grp.peer_errors(cn) == 0
    assert all(grp.member(r).get_stat(STAT_LIGHT_GRID_BUILDS) == 7 for r in range(n))
