"""Texture filtering (ST_OPT_TEXTURE_FILTER): the oracle extension's mip chains against a numpy restatement, the purpose of the filter
on the oracle, the extension's deliberate mistakes, and the CUDA path against that extension (pool and table, the level of detail's
log2, every camera buffer of the strict tier, the product tier, the option's selection, normal maps together with the filter, row
strips)."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle_texfilter import pyoracle_texfilter as T
from tests import ref64_texfilter as R
from tests.util import CAMERA_BUFFERS, assert_bits_equal, rel_l2

OPT_TEXTURE_FILTER, STAT_TEXTURE_MIP_BUILDS, OPT_NORMAL_MAPS = 17, 11, 14


def _lut_from(eo):
    """The engine's sRGB table (the one atlas_fetch decodes with), as the oracle holds it."""
    return eo.srgb_lut()


def _numpy_pool(images_in_order, lut):
    mid = ((lut[:-1] + lut[1:]).astype(np.float32) * np.float32(0.5)).astype(np.float32)
    chunks = []
    for img in images_in_order:
        cur = img
        while cur.shape[0] > 1 or cur.shape[1] > 1:
            cur = R.numpy_level(cur, lut, mid)
            chunks.append(cur.reshape(-1, 4))
    return np.concatenate(chunks) if chunks else np.zeros((0, 4), np.uint8)


def _texf_oracle(blue_noise, scene, on=True, mutation=None):
    eo = T.TextureFilterOracleEngine(blue_noise=blue_noise, mutation=mutation)
    eo.set_texture_filter(on)
    return eo, scenes.apply(eo, scene)


def _odd_sizes_scene():
    """A textured_room whose floor and fence carry images of 1x1, 1xN, Nx1 and odd sizes."""
    sc = scenes.textured_room(48, 32)
    rng = np.random.RandomState(9)
    extra = {730: (1, 1), 731: (1, 37), 732: (29, 1), 733: (13, 7), 734: (3, 65)}
    for hnd, (h, w) in extra.items():
        sc["images"][hnd] = rng.randint(0, 256, size=(h, w, 4)).astype(np.uint8)
    sc["material_textures"][100] = dict(base_color=733, emissive=731)
    sc["material_textures"][101] = dict(base_color=732, metallic_roughness=734)
    sc["material_textures"][103] = dict(emissive=730)
    return sc


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["textured_room", "demo_level", "odd_sizes"])
def test_oracle_mips_match_numpy(blue_noise, name):
    """The extension's pool is the numpy restatement's byte for byte (levels 1.. of every image, in insertion order), and its table
    points each textured slot at its image's level 1 with the image's level count."""
    sc = _odd_sizes_scene() if name == "odd_sizes" else getattr(scenes, name)(48, 32)
    eo, _ = _texf_oracle(blue_noise, sc)
    eo.tick()
    table, pool = T.parse(eo.read_texture_mips())
    imgs = list(sc["images"].values())
    want = _numpy_pool(imgs, _lut_from(eo))
    assert pool.shape == want.shape and (pool == want).all(), name
    offs, total = {}, 0
    for hnd, img in sc["images"].items():
        h, w = img.shape[:2]
        levels = 1 + int(math.floor(math.log2(max(h, w))))
        offs[hnd] = (total, levels)
        while h > 1 or w > 1:
            h, w = max(1, h >> 1), max(1, w >> 1); total += h * w
    mats = list(sc["materials"])
    for mh, tex in sc["material_textures"].items():
        for slot, key in enumerate(("base_color", "emissive", "metallic_roughness")):
            if key in tex:
                assert tuple(table[mats.index(mh), slot]) == offs[tex[key]], (name, mh, key)


def test_oracle_option_without_colour_textures_changes_nothing(blue_noise):
    """Cornell and stress_lights have no colour texture: with the option on, every buffer of the extension is the plain oracle's."""
    for sc in (scenes.cornell(64, 48), scenes.stress_lights(64, 48)):
        on, con = _texf_oracle(blue_noise, sc)
        off, coff = _texf_oracle(blue_noise, sc, on=False)
        for f in range(3):
            for e, cam in ((on, con), (off, coff)):
                e.tick(); e.render_camera(cam)
            for name in CAMERA_BUFFERS:
                assert_bits_equal(on.read_buffer(con, name), off.read_buffer(coff, name), f"{sc['name']} frame {f + 1} {name}")


def _base_colour(e, cam, w, h):
    """Linear base colour of the primary hits (G-buffer d1.w bytes, GBufferEntry::unpack's gamma 2.2) and the hit mask."""
    d0 = e.read_buffer(cam, "prim_gbuffer_d0_b").reshape(h, w, 4)
    d1 = e.read_buffer(cam, "prim_gbuffer_d1_b").reshape(h, w, 4)[..., 3].copy().view(np.uint32)
    rgb = np.stack([((d1 >> (8 * k)) & 0xff).astype(np.float64) / 255.0 for k in range(3)], -1) ** 2.2
    return rgb, d0[..., 0] != 0.0


def _primary_only(e, cam):
    e.tick()
    e.render_range(cam, 0, 0)   # K0 only


def test_filter_is_closer_to_supersampled_truth(blue_noise):
    """The purpose, on the oracle: at 96x54 the option-on primary base colour is closer (mean absolute error over pixels whose
    8x8 block is fully covered) to an 8x8-supersampled option-off base colour, box-averaged in linear light, than the option-off one:
    measured 0.360 times its error, pinned at 0.45."""
    w, h, s = 96, 54, 8
    sc = scenes.tiled_ground(w, h)
    res = {}
    for on in (False, True):
        eo, cam = _texf_oracle(blue_noise, sc, on=on)
        _primary_only(eo, cam)
        res[on] = _base_colour(eo, cam, w, h)
    big = scenes.tiled_ground(w * s, h * s)
    eb, cb = _texf_oracle(blue_noise, big, on=False)
    _primary_only(eb, cb)
    rgb, hit = _base_colour(eb, cb, w * s, h * s)
    truth = rgb.reshape(h, s, w, s, 3).mean((1, 3))
    full = hit.reshape(h, s, w, s).all((1, 3)) & res[False][1] & res[True][1]
    err = {on: float(np.abs(res[on][0][full] - truth[full]).mean()) for on in (False, True)}
    print(f"mean |base colour - 8x8 supersampled|: filter off {err[False]:.5f}, on {err[True]:.5f}, ratio {err[True] / err[False]:.3f}")
    assert full.sum() > 2000
    assert err[True] < 0.45 * err[False], err   # measured 0.360 (0.0557 against 0.1546)


P_PRIM_GBUFFER, P_GI_SAMPLING_A, P_REF_SHADING = 0, 8, 22


def _probe_frames(blue_noise, name, mutation=None, frames=2):
    """{pass: [probe records]} of the extension over `frames` Image-mode frames (K0 and K12 after the step) and one Reference-mode
    frame at depth 2 (K2 before each bounce), at 96x54; and the float64 restatement of the scene."""
    out = {P_PRIM_GBUFFER: [], P_GI_SAMPLING_A: [], P_REF_SHADING: []}
    for mode, ref_depth in ((scenes.MODE_IMAGE, 1), (scenes.MODE_REFERENCE, 2)):
        sc = getattr(scenes, name)(96, 54, mode=mode)
        sc["camera"] = dict(sc["camera"], ref_depth=ref_depth)
        eo, cam = _texf_oracle(blue_noise, sc, mutation=mutation)
        for f in range(frames if mode == scenes.MODE_IMAGE else 1):
            eo.tick()
            sched = eo.frame_schedule(cam)
            for i, p in enumerate(sched):
                is_k2 = p == P_REF_SHADING and i + 1 < len(sched) and sched[i + 1] != T.P_COMPOSITION
                if is_k2:
                    out[p].append(eo.probe(cam, p, sched[:i].count(P_REF_SHADING)))
                eo.render_range(cam, i, i)
                if p in (P_PRIM_GBUFFER, P_GI_SAMPLING_A):
                    out[p].append(eo.probe(cam, p))
        rest = R.Restatement(sc, eo.read_scene("triangles"), eo.read_scene("materials"), eo.srgb_lut())
    return {p: np.concatenate(v) for p, v in out.items()}, rest


@pytest.mark.parametrize("name", ["tiled_ground", "textured_room", "demo_level"])
def test_oracle_material_terms_inside_float64_bound(blue_noise, name):
    """The extension's filtered base colour, emissive and metallic-roughness at K0, and base colour and emissive at K12 (GI bounce
    hits) and K2 (Reference mode, depth 0..2), lie inside the float64 restatement's bound wherever the level and texel choices are
    decided; the undecided fraction is reported and kept small."""
    recs, rest = _probe_frames(blue_noise, name)
    for p, slots in ((P_PRIM_GBUFFER, (0, 1, 2)), (P_GI_SAMPLING_A, (0, 1)), (P_REF_SHADING, (0, 1))):
        stats = R.check(rest, recs[p], slots)
        frac = stats["undecided"] / max(1, stats["checked"] + stats["undecided"])
        print(f"{name} pass {p}: {stats}, undecided fraction {frac:.2e}")
        assert stats["hits"] > 200 and stats["checked"] > 400, (p, stats)
        assert frac < 0.01, (p, stats)


@pytest.mark.parametrize("mutation", sorted(T.MUTATIONS))
def test_oracle_mutation_leaves_float64_bound(blue_noise, mutation):
    """Each deliberate mistake - mips averaged on the raw bytes, no |n.d| term, taps clamped into the atlas instead of wrapped in the
    image, no half-texel centre, level weights swapped - puts material terms outside the float64 bound at K0, at the GI bounce (K12)
    and in Reference mode (K2) of tiled_ground."""
    recs, rest = _probe_frames(blue_noise, "tiled_ground", mutation=mutation)
    for p, slots in ((P_PRIM_GBUFFER, (0, 1, 2)), (P_GI_SAMPLING_A, (0, 1)), (P_REF_SHADING, (0, 1))):
        with pytest.raises(AssertionError, match="outside the float64 bound"):
            R.check(rest, recs[p], slots)


def test_log2_matches_float64():
    """The level of detail's log2 lies within 2^-21 (1 + |log2 x|) of float64 over normal and subnormal inputs."""
    rng = np.random.RandomState(1)
    x = np.concatenate([np.exp2(rng.uniform(-149, 127, 200000)), rng.uniform(0.5, 2.0, 100000), [1.0, 2.0, 0.5, 1e-45, 3.4e38]]).astype(np.float32)
    x = x[(x > 0) & np.isfinite(x)]
    got = T.log2_lod(x).astype(np.float64)
    ref = np.log2(x.astype(np.float64))
    assert (np.abs(got - ref) <= 2.0 ** -21 * (1.0 + np.abs(ref))).all()


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu_engine(blue_noise, exact, texture_filter=True, fused=None, normal_maps=False):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    e.set_option(OPT_TEXTURE_FILTER, int(texture_filter))
    if normal_maps:
        e.set_option(OPT_NORMAL_MAPS, 1)
    if fused is not None:
        from strolle_b200.engine import OPT_FUSED_PASSES
        e.set_option(OPT_FUSED_PASSES, int(fused))
    return e


MOVING = {"tiled_ground": 313, "textured_room": 304, "demo_level": None}


def _scene(name, w, h, **kw):
    return getattr(scenes, name)(w, h, **kw)


def _step(engines, scene, f, w, h):
    """Frame f: the camera drifts and turns; in tiled_ground and textured_room the box moves too."""
    c = scene["camera"]
    t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
    t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
    inst = MOVING.get(scene["name"])
    for e, cam in engines:
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t.reshape(-1), c["projection"])
        if inst is not None:
            _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == inst)
            xf = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.03 * f, 0.0, 0.02 * f], np.float32)
            e.insert_instance(inst, mesh, mat, xf)
        e.tick(); e.render_camera(cam)


@pytest.mark.gpu
def test_device_pool_matches_oracle(blue_noise):
    """st_read_scene("texture_mips") equals the extension's pool and table byte for byte after an insert, a re-insert with new
    pixels, a removal, and the option switching off and on; the builds are counted."""
    sc = scenes.textured_room(64, 36)
    eg = _gpu_engine(blue_noise, True)
    eo, _ = _texf_oracle(blue_noise, sc)
    scenes.apply(eg, sc)
    rng = np.random.RandomState(4)
    def same(what):
        assert_bits_equal(eg.read_scene("texture_mips").view(np.uint32), eo.read_texture_mips(), what)
    for e in (eg, eo):
        e.tick()
    same("insert")
    new = rng.randint(0, 256, size=(64, 64, 4)).astype(np.uint8)
    for e in (eg, eo):
        e.insert_image(700, new); e.tick()
    same("re-insert")
    for e in (eg, eo):
        e.remove_image(702); e.tick()
    same("removal")
    eg.set_option(OPT_TEXTURE_FILTER, 0); eg.tick()
    with pytest.raises(Exception):
        eg.read_scene("texture_mips")
    eg.set_option(OPT_TEXTURE_FILTER, 1); eg.tick()
    same("off, then on")
    assert eg.get_stat(STAT_TEXTURE_MIP_BUILDS) == 4


@pytest.mark.gpu
def test_device_log2_matches_oracle(blue_noise):
    """st_device_math op 7 is the oracle's log2 bit for bit, and within its bound of float64."""
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise)
    rng = np.random.RandomState(2)
    x = np.concatenate([np.exp2(rng.uniform(-149, 127, 200000)), rng.uniform(0.5, 2.0, 100000)]).astype(np.float32)
    x = x[(x > 0) & np.isfinite(x)]
    got = e.device_math("log2_lod", x)
    assert_bits_equal(got, T.log2_lod(x), "log2")
    ref = np.log2(x.astype(np.float64))
    assert (np.abs(got.astype(np.float64) - ref) <= 2.0 ** -21 * (1.0 + np.abs(ref))).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiled_ground", "textured_room", "demo_level"])
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
@pytest.mark.parametrize("fused", [False, True])
def test_strict_tier_bit_exact_with_oracle(oracle, blue_noise, name, size, fused):
    """Option on, strict arithmetic, 13 frames with the camera (and an instance) moving: every camera buffer is the extension's,
    bit for bit (the fused schedule: every buffer it still writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = size
    scene = _scene(name, w, h)
    eg = _gpu_engine(blue_noise, True, fused=fused)
    cg = scenes.apply(eg, scene)
    eo, co = _texf_oracle(blue_noise, scene)
    names = [n for n in CAMERA_BUFFERS if not (fused and n in NOT_WRITTEN_WHEN_FUSED)]
    for f in range(13):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for n in names:
            assert_bits_equal(eg.read_buffer(cg, n), eo.read_buffer(co, n), f"{name} fused={fused} {size} frame {f + 1} {n}")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2])
def test_reference_mode_bit_exact_with_oracle(oracle, blue_noise, depth):
    """Reference mode with the option on: every camera buffer (K1's hits, K2's filtered shading at every depth, the accumulated
    colours, the output) is the extension's, bit for bit, over 13 moving frames."""
    w, h = 224, 126
    scene = scenes.tiled_ground(w, h, mode=scenes.MODE_REFERENCE, ref_depth=depth)
    eg = _gpu_engine(blue_noise, True)
    cg = scenes.apply(eg, scene)
    eo, co = _texf_oracle(blue_noise, scene)
    for f in range(13):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for n in CAMERA_BUFFERS:
            assert_bits_equal(eg.read_buffer(cg, n), eo.read_buffer(co, n), f"depth {depth} frame {f + 1} {n}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,bound", [("tiled_ground", 1e-3), ("demo_level", 1e-3), ("textured_room", 2e-2)])
def test_product_tier_within_tolerance_of_oracle(oracle, blue_noise, name, bound):
    """Option on, product defaults: the G-buffer is the strict tier's bit for bit, and the composed frame stays within the bound
    (relative per-channel L2) of the extension over 13 frames."""
    w, h = 224, 126
    scene = _scene(name, w, h)
    prod, strict = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, True)
    cp, cs = scenes.apply(prod, scene), scenes.apply(strict, scene)
    eo, co = _texf_oracle(blue_noise, scene)
    worst = 0.0
    for f in range(13):
        for e, cam in ((prod, cp), (strict, cs), (eo, co)):
            e.tick(); e.render_camera(cam)
        for n in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "prim_surface_map_a",
                  "prim_surface_map_b", "surface_nd", "prim_triangle_ids"):
            assert_bits_equal(prod.read_buffer(cp, n), strict.read_buffer(cs, n), f"frame {f + 1} {n}")
        a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
        b = eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
        for ch in range(3):
            worst = max(worst, rel_l2(a[:, ch], b[:, ch]))
    print(f"{name}: worst relative L2 {worst:.3g}")
    assert worst <= bound


@pytest.mark.gpu
def test_option_selection(blue_noise):
    """Cornell (no texture) is bit-identical with the option on and off; on textured scenes the triangle ids are identical; any
    value but 0 and 1 is refused."""
    import strolle_b200
    w, h = 96, 64
    for sc, all_buffers in ((scenes.cornell(w, h), True), (scenes.tiled_ground(w, h), False), (scenes.demo_level(w, h), False)):
        on, off = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, False, texture_filter=False)
        con, coff = scenes.apply(on, sc), scenes.apply(off, sc)
        for f in range(5):
            for e, cam in ((on, con), (off, coff)):
                e.tick(); e.render_camera(cam)
            for n in (CAMERA_BUFFERS if all_buffers else ("prim_triangle_ids",)):
                assert_bits_equal(on.read_buffer(con, n), off.read_buffer(coff, n), f"{sc['name']} frame {f + 1} {n}")
    e = strolle_b200.Engine(blue_noise=blue_noise)
    for bad in (-1, 2, 17):
        with pytest.raises(Exception):
            e.set_option(OPT_TEXTURE_FILTER, bad)


@pytest.mark.gpu
def test_with_normal_maps(blue_noise):
    """Both options on: the normals are those of the normal-maps-only run, the base colours those of the filter-only run."""
    w, h = 224, 126
    sc = scenes.normal_mapped_room(w, h)
    sc["material_textures"] = {k: dict(v) for k, v in sc["material_textures"].items()}
    sc["images"] = dict(sc["images"])
    sc["images"][715] = np.random.RandomState(8).randint(0, 256, size=(40, 24, 4)).astype(np.uint8)
    for k in sc["material_textures"]:
        sc["material_textures"][k]["base_color"] = 715
    both = _gpu_engine(blue_noise, True, normal_maps=True)
    nm = _gpu_engine(blue_noise, True, texture_filter=False, normal_maps=True)
    tf = _gpu_engine(blue_noise, True)
    cams = [scenes.apply(e, sc) for e in (both, nm, tf)]
    for e, cam in zip((both, nm, tf), cams):
        e.tick(); e.render_camera(cam)
    g = [e.read_buffer(c, "prim_gbuffer_d0_b").reshape(h, w, 4) for e, c in zip((both, nm, tf), cams)]
    d = [e.read_buffer(c, "prim_gbuffer_d1_b").reshape(h, w, 4) for e, c in zip((both, nm, tf), cams)]
    assert_bits_equal(g[0][..., 1:3], g[1][..., 1:3], "normals")
    assert_bits_equal(d[0][..., 3], d[2][..., 3], "base colours")
    assert (d[0][..., 3].view(np.uint32) != d[1][..., 3].view(np.uint32)).sum() > 1000


def _devices(n):
    import torch
    have = max(torch.cuda.device_count(), 1)
    return [k % have for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,size", [(2, (320, 288)), (3, (256, 400))])
def test_row_strips_match_single_gpu(blue_noise, n, size):
    """Option on, tiled_ground as n row strips (st_multi_*, devices reused when there are fewer), camera and box moving: every
    camera buffer is the single-GPU frame's, bit for bit, over 7 frames."""
    import strolle_b200
    w, h = size
    scene = scenes.tiled_ground(w, h)
    one = _gpu_engine(blue_noise, False)
    grp = strolle_b200.MultiEngine(_devices(n), blue_noise=blue_noise)
    grp.set_option(OPT_TEXTURE_FILTER, 1)
    c1, cn = scenes.apply(one, scene), scenes.apply(grp, scene)
    for f in range(7):
        _step([(one, c1), (grp, cn)], scene, f, w, h)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(cn, name), one.read_buffer(c1, name), f"{n} strips frame {f + 1} {name}")
    assert grp.peer_errors(cn) == 0
