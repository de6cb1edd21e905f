"""Normal maps (ST_OPT_NORMAL_MAPS): the oracle's restatement of the rule (oracle_nmap/) against the float64 restatement
(tests/ref64_normalmap.py), the CUDA path against that oracle frame by frame, the option's selection, the two arithmetic tiers, the
fused schedule and row strips."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle_nmap import pyoracle_nmap
from tests import ref64_normalmap as R
from tests.util import CAMERA_BUFFERS, Frame, assert_bits_equal, rel_l2

OPT_NORMAL_MAPS, STAT_NORMAL_MAP_LAUNCHES = 14, 8
TORUS = 304   # the instance normal_mapped_room's tests move


def _restatement_inputs(e, scene):
    tri, mats, bvh = e.read_scene("triangles"), e.read_scene("materials"), e.read_scene("bvh")
    return tri, R.material_of_triangles(bvh, tri.size // 36), mats, R.images_by_rect(mats, scene)


def _reference(e, cam, scene, w, h, **kw):
    tri, mt, mats, imgs = _restatement_inputs(e, scene)
    tid = e.read_buffer(cam, "prim_triangle_ids").reshape(h, w, 4)[..., 0]
    return R.evaluate(tri, mt, mats, imgs, e.read_buffer(cam, "curr_camera"), tid, w, h, **kw)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_quad_default_keeps_zero_tangents():
    """`_quad` without `tangents` builds the same bytes as before the argument existed: zero tangents."""
    q = np.stack(scenes._quad((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1)))
    assert (q[:, 24:36] == 0).all()
    for name in ("textured_room", "cornell"):
        s = getattr(scenes, name)(32, 32)
        assert all((m[:, 24:36] == 0).all() for m in s["meshes"].values()), name


def test_scene_covers_every_case(oracle, blue_noise):
    """normal_mapped_room has a mapped floor and wall, a tangent torus and a mirrored copy, a two-sided panel seen from behind,
    a mapped mesh without tangents and an unmapped material, all dielectric with perceptual roughness >= 0.5 - and each is on screen."""
    sc = scenes.normal_mapped_room(224, 126)
    for params, _ in sc["materials"].values():
        assert params[9] == 0.0 and params[8] >= 0.5
    xf = {h: np.asarray(x, np.float64).reshape(4, 3) for h, _, _, x in sc["instances"]}
    assert np.linalg.det(xf[305][:3]) < 0 < np.linalg.det(xf[304][:3])
    assert (sc["meshes"][203][:, 24:36] == 0).all() and sc["material_textures"][101]["normal_map"] == 710
    assert 103 not in sc["material_textures"]
    eo = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(eo, sc)
    eo.tick(); eo.render_camera(cam)
    ref = _reference(eo, cam, sc, 224, 126)
    assert (ref["hit"] & (ref["sign"] < 0)).sum() > 500, "back faces on screen (the panel)"
    assert ref["fallback"].sum() > 200, "fallback pixels on screen (the mesh without tangents, the below-surface patch)"
    assert (ref["hit"] & ~ref["mapped"]).sum() > 100, "unmapped material on screen"


def test_restatement_interpolated_normal_matches_oracle(oracle, blue_noise):
    """With every map removed, the restatement's N is what the oracle (bit-exact with the kernels) stores in the surface map:
    the float64 camera rays, barycentrics and the bound's interpolation terms are right."""
    sc = scenes.normal_mapped_room(224, 126)
    eo = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(eo, sc)
    eo.tick(); eo.render_camera(cam)
    tri, mt, mats, _ = _restatement_inputs(eo, sc)
    mats = mats.reshape(-1, 28).copy(); mats[:, 24:28] = 0
    tid = eo.read_buffer(cam, "prim_triangle_ids").reshape(126, 224, 4)[..., 0]
    ref = R.evaluate(tri, mt, mats, {}, eo.read_buffer(cam, "curr_camera"), tid, 224, 126)
    surf = eo.read_buffer(cam, "prim_surface_map_b").reshape(126, 224, 4)   # frame 1 writes slot 1
    got = R.oct_decode(surf[..., :2])
    stats = R.check(got, ref)
    assert stats["pixels"] > 20000 and stats["worst_ratio"] < 0.5, stats


def _nmap_oracle(blue_noise, scene, on=True, mutation=None):
    eo = pyoracle_nmap.NormalMapOracleEngine(blue_noise=blue_noise, mutation=mutation)
    eo.set_normal_maps(on)
    return eo, scenes.apply(eo, scene)


def test_oracle_normals_inside_float64_bound(oracle, blue_noise):
    """The oracle with the option on: its surface-map normals lie inside the float64 bound of the rule (the texel choice and the
    n'.N test taken either way only inside their derived margins); on the mesh without tangents and on the unmapped material every
    G-buffer word is the option-off oracle's."""
    sc = scenes.normal_mapped_room(224, 126)
    eo, c = _nmap_oracle(blue_noise, sc)
    off, coff = _nmap_oracle(blue_noise, sc, on=False)
    for e, cam in ((eo, c), (off, coff)):
        e.tick(); e.render_camera(cam)
    ref = _reference(eo, c, sc, 224, 126)
    stats = R.check(R.oct_decode(eo.read_buffer(c, "prim_surface_map_b").reshape(126, 224, 4)[..., :2]), ref)
    assert stats["mapped"] > 20000 and stats["unknown"] < 20 and stats["fallback"] > 200, stats
    tri = eo.read_scene("triangles").reshape(-1, 9, 4)
    tid = eo.read_buffer(c, "prim_triangle_ids").reshape(126, 224, 4)[..., 0].view(np.uint32)
    same = ref["hit"] & (~ref["mapped"] | np.isnan(tri[np.where(ref["hit"], tid, 0), 2, 0]))
    assert same.sum() > 300
    for name in ("prim_gbuffer_d0_b", "prim_gbuffer_d1_b", "prim_surface_map_b"):
        a = eo.read_buffer(c, name).reshape(126, 224, 4)[same]
        b = off.read_buffer(coff, name).reshape(126, 224, 4)[same]
        assert_bits_equal(a, b, name)


@pytest.mark.parametrize("mutation", sorted(pyoracle_nmap.MUTATIONS))
def test_oracle_mutation_fails_float64_check(blue_noise, mutation):
    """Each deliberate mistake in the oracle's rule - sRGB decode of the texel, B = w (T x N), no back-face sign, T renormalised,
    no fallback - puts its normals outside the float64 bound."""
    sc = scenes.normal_mapped_room(224, 126)
    eo, c = _nmap_oracle(blue_noise, sc, mutation=mutation)
    eo.tick(); eo.render_camera(c)
    ref = _reference(eo, c, sc, 224, 126)
    with pytest.raises(AssertionError, match="outside the float64 bound"):
        R.check(R.oct_decode(eo.read_buffer(c, "prim_surface_map_b").reshape(126, 224, 4)[..., :2]), ref)


def test_oracle_option_without_maps_changes_nothing(blue_noise):
    """Cornell has no normal map: with the option on, the oracle's buffers are bit-identical to the option off, 7 frames."""
    sc = scenes.cornell(96, 64)
    on, con = _nmap_oracle(blue_noise, sc)
    off, coff = _nmap_oracle(blue_noise, sc, on=False)
    for f in range(7):
        for e, cam in ((on, con), (off, coff)):
            e.tick(); e.render_camera(cam)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(on.read_buffer(con, name), off.read_buffer(coff, name), f"frame {f + 1} {name}")


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu_engine(blue_noise, exact, normal_maps=True, fused=None):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    e.set_option(OPT_NORMAL_MAPS, int(normal_maps))
    if fused is not None:
        from strolle_b200.engine import OPT_FUSED_PASSES
        e.set_option(OPT_FUSED_PASSES, int(fused))
    return e


def _move(f, scene, w, h):
    """Frame f's camera transform and torus affine: both drift, the torus also turns."""
    eye = (0.4 + 0.03 * f, 1.5 - 0.02 * f, 3.8 - 0.04 * f)
    cam = scenes.look_at_transform(eye, (0.0, 0.6, -0.5))
    a = 0.08 * f
    c, s = math.cos(a), math.sin(a)
    xf = np.array([c, 0, -s, s, 0, c, 0, -1, 0, -0.3 + 0.02 * f, 0.7, -0.6], np.float32)
    return cam, xf


def _step(engines, scene, f, w, h):
    c = scene["camera"]
    t, xf = _move(f, scene, w, h)
    _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == TORUS)
    for e, cam in engines:
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t, c["projection"])
        e.insert_instance(TORUS, mesh, mat, xf)
        e.tick(); e.render_camera(cam)


def _device_normals(e, cam, w, h):
    """The shading normal as each G-buffer consumer sees it: surface_nd, the surface map and the G-buffer d0 (this frame's slot)."""
    cur = "b" if (e.frame() - 1) % 2 == 1 else "a"
    nd = e.read_buffer(cam, "surface_nd").reshape(h, w, 4)[..., :3]
    surf = R.oct_decode(e.read_buffer(cam, "prim_surface_map_" + cur).reshape(h, w, 4)[..., :2])
    g0 = R.oct_decode(e.read_buffer(cam, "prim_gbuffer_d0_" + cur).reshape(h, w, 4)[..., 1:3])
    return nd, surf, g0


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
@pytest.mark.parametrize("exact", [True, False])
def test_device_normals_inside_float64_bound(blue_noise, size, exact):
    """13 frames, camera and torus moving: every primary-hit normal (surface_nd, surface map, G-buffer) lies inside the float64
    bound of the rule, in the strict and in the product tier; on the mesh without tangents and on the unmapped material it is
    bit-identical to the same frame with the option off."""
    w, h = size
    scene = scenes.normal_mapped_room(w, h)
    on, off = _gpu_engine(blue_noise, exact), _gpu_engine(blue_noise, exact, normal_maps=False)
    con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
    total = dict(pixels=0, mapped=0, fallback=0, texel_margin=0, fallback_margin=0, took_alt=0, unknown=0)
    for f in range(13):
        _step([(on, con), (off, coff)], scene, f, w, h)
        assert_bits_equal(on.read_buffer(con, "prim_triangle_ids"), off.read_buffer(coff, "prim_triangle_ids"), f"frame {f + 1} triangle ids")
        ref = _reference(on, con, scene, w, h)
        for what, got in zip(("surface_nd", "surface map", "G-buffer"), _device_normals(on, con, w, h)):
            try:
                stats = R.check(got, ref)
            except AssertionError as err:
                raise AssertionError(f"frame {f + 1} {what}: {err}")
        for k in total:
            total[k] += stats[k]
        nd_on = on.read_buffer(con, "surface_nd").reshape(h, w, 4)
        nd_off = off.read_buffer(coff, "surface_nd").reshape(h, w, 4)
        assert_bits_equal(nd_on[~ref["mapped"]], nd_off[~ref["mapped"]], f"frame {f + 1} unmapped pixels")
    assert total["mapped"] > 0.5 * total["pixels"] and total["fallback"] > 0, total
    assert total["texel_margin"] + total["fallback_margin"] < 0.03 * total["pixels"], total
    assert total["unknown"] <= 0.001 * total["pixels"], total   # uv on the edge of an image's rect: not checked, so kept rare


@pytest.mark.gpu
def test_mesh_without_tangents_keeps_interpolated_normal(blue_noise):
    """The brick-mapped box has no tangents (baked NaN): with the option on its pixels are bit-identical to the option off."""
    w, h = 224, 126
    scene = scenes.normal_mapped_room(w, h)
    on, off = _gpu_engine(blue_noise, True), _gpu_engine(blue_noise, True, normal_maps=False)
    con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
    on.tick(); off.tick(); on.render_camera(con); off.render_camera(coff)
    tri = on.read_scene("triangles").reshape(-1, 9, 4)
    tid = on.read_buffer(con, "prim_triangle_ids").reshape(h, w, 4)[..., 0].view(np.uint32)
    hit = tid != 0xffffffff
    no_tangent = np.zeros((h, w), bool)
    no_tangent[hit] = np.isnan(tri[tid[hit], 2, 0])
    assert no_tangent.sum() > 200
    for name in ("surface_nd", "prim_gbuffer_d0_b", "prim_surface_map_b"):
        a = on.read_buffer(con, name).reshape(h, w, 4)[no_tangent]
        b = off.read_buffer(coff, name).reshape(h, w, 4)[no_tangent]
        assert_bits_equal(a, b, name)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
@pytest.mark.parametrize("fused", [False, True])
def test_strict_tier_bit_exact_with_oracle(oracle, blue_noise, size, fused):
    """Option on, strict arithmetic, 13 frames with the camera and the torus moving: every camera buffer - G-buffer, GI bounce hits,
    reservoirs, SVGF, output - is the normal-mapped oracle's, bit for bit (the fused schedule: every buffer it still writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = size
    scene = scenes.normal_mapped_room(w, h)
    eg = _gpu_engine(blue_noise, True, fused=fused)
    cg = scenes.apply(eg, scene)
    eo, co = _nmap_oracle(blue_noise, scene)
    names = [n for n in CAMERA_BUFFERS if not (fused and n in NOT_WRITTEN_WHEN_FUSED)]
    for f in range(13):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for name in names:
            assert_bits_equal(eg.read_buffer(cg, name), eo.read_buffer(co, name), f"fused={fused} {size} frame {f + 1} {name}")
    assert eg.get_stat(STAT_NORMAL_MAP_LAUNCHES) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2])
def test_reference_mode_bit_exact_with_oracle(oracle, blue_noise, depth):
    """Reference mode with the option on: K1's packed hits at every depth (bounce hits included), K2's shading and nudge along
    the mapped normal and the accumulated colours are the normal-mapped oracle's, bit for bit, over 5 moving frames."""
    w, h = 224, 126
    scene = scenes.normal_mapped_room(w, h, mode=scenes.MODE_REFERENCE, ref_depth=depth)
    eg = _gpu_engine(blue_noise, True)
    cg = scenes.apply(eg, scene)
    eo, co = _nmap_oracle(blue_noise, scene)
    for f in range(5):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for name in ("ref_hits", "ref_rays", "ref_colors", "output"):
            assert_bits_equal(eg.read_buffer(cg, name), eo.read_buffer(co, name), f"depth {depth} frame {f + 1} {name}")
    assert eg.get_stat(STAT_NORMAL_MAP_LAUNCHES) == 5 * (depth + 1)


@pytest.mark.gpu
def test_product_tier_within_tolerance_of_oracle(oracle, blue_noise):
    """Option on, product defaults: the G-buffer, surface maps, surface_nd and triangle ids are the strict tier's bit for bit, and
    the composed frame stays within 1e-3 relative per-channel L2 of the normal-mapped oracle over 13 frames."""
    w, h = 224, 126
    scene = scenes.normal_mapped_room(w, h)
    prod, strict = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, True)
    cp, cs = scenes.apply(prod, scene), scenes.apply(strict, scene)
    eo, co = _nmap_oracle(blue_noise, scene)
    for f in range(13):
        for e, cam in ((prod, cp), (strict, cs), (eo, co)):
            e.tick(); e.render_camera(cam)
        for name in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "prim_surface_map_a",
                     "prim_surface_map_b", "surface_nd", "prim_triangle_ids"):
            assert_bits_equal(prod.read_buffer(cp, name), strict.read_buffer(cs, name), f"frame {f + 1} {name}")
        a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
        b = eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
        for ch in range(3):
            assert rel_l2(a[:, ch], b[:, ch]) <= 1e-3, f"frame {f + 1} channel {ch}"


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
def test_fused_schedule_matches_unfused(blue_noise, size):
    """Option on, strict arithmetic: the fused schedule (K12 + K13 in one launch, the NMAP instantiation of k_gi_sampling_fused)
    gives the reservoirs, samples and frame of the one-launch-per-pass schedule over 13 moving frames."""
    w, h = size
    scene = scenes.normal_mapped_room(w, h)
    a, b = _gpu_engine(blue_noise, True, fused=False), _gpu_engine(blue_noise, True, fused=True)
    ca, cb = scenes.apply(a, scene), scenes.apply(b, scene)
    for f in range(13):
        _step([(a, ca), (b, cb)], scene, f, w, h)
        for name in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "surface_nd", "di_reservoirs_0", "gi_reservoirs_0", "di_diff_curr_colors",
                     "gi_diff_curr_colors", "di_diff_moments_a", "gi_diff_moments_b", "output"):
            assert_bits_equal(b.read_buffer(cb, name), a.read_buffer(ca, name), f"frame {f + 1} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [1, 2])
def test_reference_mode_hits_use_mapped_normal(blue_noise, depth):
    """Reference mode: the camera-ray hits K1 packs (ref_hits) carry the mapped normal, inside the float64 bound; the frame
    converges to finite colours."""
    w, h = 224, 126
    scene = scenes.normal_mapped_room(w, h, mode=scenes.MODE_REFERENCE, ref_depth=depth)
    e = _gpu_engine(blue_noise, True)
    g = _gpu_engine(blue_noise, True)   # an Image-mode camera gives prim_triangle_ids for the same rays
    cam = scenes.apply(e, scene)
    img_scene = scenes.normal_mapped_room(w, h)
    cg = scenes.apply(g, img_scene)
    e.tick(); g.tick(); g.render_camera(cg)
    fr = Frame(e, cam, w, h)
    fr.run_to(fr.steps(21)[0])   # P_REF_TRACING, depth 0
    hits = e.read_buffer(cam, "ref_hits").reshape(h, w, 2, 4)
    got = R.oct_decode(hits[:, :, 1, :2])
    ref = _reference(g, cg, img_scene, w, h)
    stats = R.check(got, ref)
    assert stats["mapped"] > 20000, stats
    fr.run_to(len(fr.sched) - 1)
    for _ in range(3):
        e.tick(); e.render_camera(cam)
    out = e.read_buffer(cam, "output").reshape(h, w, 4)
    assert np.isfinite(out).all() and out[..., :3].mean() > 0.0
    assert e.get_stat(STAT_NORMAL_MAP_LAUNCHES) == 4 * (depth + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name", ["cornell", "dungeon"])
def test_option_without_maps_changes_nothing(blue_noise, scene_name):
    """Scenes without normal maps: the option on is bit-identical to the option off in every camera buffer, and no NMAP kernel
    runs; Image and Reference mode, strict and product tier."""
    for exact in (True, False):
        for mode in (scenes.MODE_IMAGE, scenes.MODE_REFERENCE):
            scene = scenes.cornell(96, 64, mode=mode) if scene_name == "cornell" else scenes.dungeon(96, 64, mode=mode, cells=6)
            on, off = _gpu_engine(blue_noise, exact), _gpu_engine(blue_noise, exact, normal_maps=False)
            con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
            for f in range(7):
                on.tick(); off.tick(); on.render_camera(con); off.render_camera(coff)
                for name in CAMERA_BUFFERS:
                    assert_bits_equal(on.read_buffer(con, name), off.read_buffer(coff, name), f"{scene_name} exact={exact} mode={mode} frame {f + 1} {name}")
            assert on.get_stat(STAT_NORMAL_MAP_LAUNCHES) == 0


@pytest.mark.gpu
def test_selection_follows_option_and_materials(blue_noise):
    """The NMAP kernels run only with the option on and a normal map in the material table, decided at st_tick: the stat counts
    one G-buffer and one GI-sampling launch per tracing frame; turning the option off at a tick stops them."""
    w, h = 96, 64
    scene = scenes.normal_mapped_room(w, h)
    e = _gpu_engine(blue_noise, True, fused=True)
    cam = scenes.apply(e, scene)
    counts = []
    for f in range(6):   # one GI cycle: the G-buffer every frame, GI sampling (fused K12 + K13) on frames 2 and 4-6 of it
        e.tick(); e.render_camera(cam)
        counts.append(e.get_stat(STAT_NORMAL_MAP_LAUNCHES))
    launches = np.diff([0] + counts)
    assert (launches >= 1).all() and (launches <= 2).all() and (launches == 2).any(), launches
    e.set_option(OPT_NORMAL_MAPS, 0)
    e.tick(); e.render_camera(cam)
    assert e.get_stat(STAT_NORMAL_MAP_LAUNCHES) == counts[-1]
    e.set_option(OPT_NORMAL_MAPS, 1)
    e.tick(); e.render_camera(cam)
    assert e.get_stat(STAT_NORMAL_MAP_LAUNCHES) > counts[-1]


def _devices(n):
    import torch
    have = max(torch.cuda.device_count(), 1)
    return [k % have for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,size,dma", [(2, (320, 288), 0), (2, (320, 288), 2), (3, (256, 400), 0), (3, (256, 400), 2)])
def test_row_strips_match_single_gpu(blue_noise, n, size, dma):
    """Option on, the new scene as n row strips (st_multi_*, devices reused when there are fewer; ST_OPT_STRIP_DMA 0 = G-buffer
    halo rows recomputed by each strip with the NMAP kernel, 2 = pushed by copy engine): every camera buffer is the single-GPU
    frame's, bit for bit, over 7 moving frames."""
    import strolle_b200
    from strolle_b200.engine import OPT_STRIP_DMA
    w, h = size
    scene = scenes.normal_mapped_room(w, h)
    one = _gpu_engine(blue_noise, False)
    grp = strolle_b200.MultiEngine(_devices(n), blue_noise=blue_noise)
    grp.set_option(OPT_NORMAL_MAPS, 1)
    grp.set_option(OPT_STRIP_DMA, dma)
    c1, cn = scenes.apply(one, scene), scenes.apply(grp, scene)
    for f in range(7):
        _step([(one, c1), (grp, cn)], scene, f, w, h)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(cn, name), one.read_buffer(c1, name), f"{n} strips dma {dma} frame {f + 1} {name}")
    assert grp.peer_errors(cn) == 0
    assert all(grp.member(r).get_stat(STAT_NORMAL_MAP_LAUNCHES) > 0 for r in range(n))
