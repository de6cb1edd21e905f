"""ST_OPT_BVH_REFIT: ticks that only move instances bake their triangles on the device and refit the BVH boxes over the last
rebuild's topology.  A numpy restatement of the refit is pinned against the host builder's streams (no device), then the device
bake against the host bake, the device refit against the restatement, the rebuild budget and fallbacks against an option-off
engine, traversal against the rebuild engine, whole frames against the oracle and row strips against one GPU."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from tests.util import CAMERA_BUFFERS, assert_bits_equal, random_rays, rel_l2

OPT_BVH_REFIT, STAT_BVH_REFITS = 15, 9
F32_MAX = np.float32(3.4028234663852886e38)
BOX = 306   # the Cornell box instance the tests move


# ---- numpy restatement ----------------------------------------------------------------------------------------------------------

def _zmin(v):
    """Per-column NaN-ignoring minimum with -0 below +0 (the kernels' order-independent Box::grow); +FLT_MAX when empty."""
    if len(v) == 0:
        return np.full(3, F32_MAX, np.float32)
    m = np.nanmin(v, axis=0).astype(np.float32)
    neg0 = ((v == 0) & np.signbit(v)).any(axis=0)
    return np.where((m == 0) & neg0, np.float32(-0.0), m).astype(np.float32)


def _zmax(v):
    if len(v) == 0:
        return np.full(3, -F32_MAX, np.float32)
    m = np.nanmax(v, axis=0).astype(np.float32)
    pos0 = ((v == 0) & ~np.signbit(v)).any(axis=0)
    return np.where((m == 0) & pos0, np.float32(0.0), np.where(m == 0, np.float32(-0.0), m)).astype(np.float32)


def refit_restatement(stream, triangles):
    """The refit over a flattened stream: leaf runs [flags, tri, mat, 1] give the box of their triangles' three positions, internal
    nodes (.w of their first entry 0) the union of their children's; every child box is stored into its parent's slot (lo at
    ptr / ptr + 2, hi at ptr + 1 / ptr + 3, .w kept).  Returns (refit stream, mask of the internal nodes' box floats)."""
    s = np.array(stream, np.float32).reshape(-1, 4).copy()
    bits = s.view(np.uint32)
    pos = np.asarray(triangles, np.float32).reshape(-1, 9, 4)[:, [0, 3, 6], :3]
    mask = np.zeros(s.shape, bool)
    if len(s) == 0 or bits[0, 3] == 1:
        return s, mask

    def walk(ptr):
        if bits[ptr, 3] == 0:
            llo, lhi = walk(ptr + 4)
            rlo, rhi = walk(int(bits[ptr + 1, 3]))
            s[ptr, :3], s[ptr + 1, :3], s[ptr + 2, :3], s[ptr + 3, :3] = llo, lhi, rlo, rhi
            mask[ptr:ptr + 4, :3] = True
            return _zmin(np.stack([llo, rlo])), _zmax(np.stack([lhi, rhi]))
        ids = []
        while True:
            ids.append(int(bits[ptr, 1]))
            if not bits[ptr, 0] & 1:
                break
            ptr += 1
        p = pos[ids].reshape(-1, 3)
        return _zmin(p), _zmax(p)

    walk(0)
    return s, mask


@pytest.mark.parametrize("scene_name", ["cornell", "dungeon"])
def test_restatement_reproduces_builder_stream(oracle, blue_noise, scene_name):
    """Unmoved, the restatement applied to the host builder's stream (primitives from the oracle engine's baked triangles, as
    test_bvh_builder does) gives that stream back bit for bit: it is the builder's box arithmetic, so the GPU tests can use it."""
    from strolle_b200.engine import BvhBuilder
    scene = scenes.cornell(32, 32) if scene_name == "cornell" else scenes.demo_level(32, 32, textures=False)
    eo = oracle.OracleEngine(blue_noise=blue_noise)
    scenes.apply(eo, scene)
    eo.tick()
    tris = eo.read_scene("triangles").reshape(-1, 9, 4)
    bits = eo.read_scene("bvh").reshape(-1, 4).view(np.uint32)
    leaf = bits[:, 3] == 1
    mat_of = {int(t): int(m) for t, m in zip(bits[leaf, 1], bits[leaf, 2])}
    p0, p1, p2 = tris[:, 0, :3], tris[:, 3, :3], tris[:, 6, :3]
    prims = np.zeros((len(tris), 11), np.float32)
    prims[:, 0] = np.arange(len(tris), dtype=np.uint32).view(np.float32)
    prims[:, 1] = np.array([mat_of.get(i, 0) for i in range(len(tris))], np.uint32).view(np.float32)
    prims[:, 2:5] = ((p0 + p1) + p2) / np.float32(3.0)
    prims[:, 5:8] = np.minimum(np.minimum(p0, p1), p2)
    prims[:, 8:11] = np.maximum(np.maximum(p0, p1), p2)
    stream = BvhBuilder().build(prims, reuse=False)
    got, mask = refit_restatement(stream, tris)
    assert mask.sum() > 12 * 10
    assert_bits_equal(got, stream, f"{scene_name}: restatement of the unmoved refit")


def test_restatement_moves_boxes():
    """The restatement is not the identity: translating the triangles shifts every box by the translation, .w words unchanged."""
    from strolle_b200.engine import BvhBuilder
    rng = np.random.RandomState(5)
    tris = np.zeros((200, 9, 4), np.float32)
    tris[:, [0, 3, 6], :3] = (rng.uniform(-5, 5, size=(200, 1, 3)) + rng.normal(scale=0.3, size=(200, 3, 3))).astype(np.float32)
    p = tris[:, [0, 3, 6], :3]
    prims = np.zeros((200, 11), np.float32)
    prims[:, 0] = np.arange(200, dtype=np.uint32).view(np.float32)
    prims[:, 2:5] = ((p[:, 0] + p[:, 1]) + p[:, 2]) / np.float32(3.0)
    prims[:, 5:8], prims[:, 8:11] = p.min(axis=1), p.max(axis=1)
    stream = BvhBuilder().build(prims, reuse=False)
    moved = tris.copy()
    moved[:, [0, 3, 6], :3] += np.float32(2.0)
    got, mask = refit_restatement(stream, moved)
    assert_bits_equal(got[~mask], stream[~mask], "leaf entries and .w words")
    assert np.allclose(got[mask], stream[mask] + 2.0, atol=1e-5)


# ---- GPU --------------------------------------------------------------------------------------------------------------------------

def _engine(blue_noise, exact, refit=30):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    e.set_option(OPT_BVH_REFIT, refit)
    return e


def _box_xf(scene, f):
    """Frame f's affine of the Cornell box BOX: turned about its own vertical axis and slid along x and z."""
    mesh = next(m for h, m, _, _ in scene["instances"] if h == BOX)
    c = scene["meshes"][mesh].reshape(-1, 36)[:, :9].reshape(-1, 3).mean(axis=0)
    a = 0.07 * f
    ca, sa = math.cos(a), math.sin(a)
    r = np.array([[ca, 0, sa], [0, 1, 0], [-sa, 0, ca]])   # rows: world = r @ local
    t = c - r @ c + np.array([0.015 * f, 0.0, -0.01 * f])
    return np.concatenate([r[:, 0], r[:, 1], r[:, 2], t]).astype(np.float32)


def _moves(scene_name, scene, f):
    """(instance, mesh, material, affine) re-inserted before tick f (f = 0 is the first tick: nothing moves yet)."""
    if f == 0:
        return []
    if scene_name == "cornell":
        _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == BOX)
        return [(BOX, mesh, mat, _box_xf(scene, f))]
    return scenes.demo_level_animated(0.05 * f)


def _scene(scene_name, w, h):
    return scenes.cornell(w, h) if scene_name == "cornell" else scenes.demo_level(w, h)


def _step(pairs, moves):
    for e, cam in pairs:
        for inst in moves:
            e.insert_instance(*inst)
        e.tick()
        if cam is not None:
            e.render_camera(cam)


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name", ["cornell", "dungeon"])
@pytest.mark.parametrize("exact", [True, False])
def test_device_bake_and_refit(oracle, blue_noise, scene_name, exact):
    """13 ticks with the box moving / the tori turning: after every tick the device's triangle array is the oracle's (which rebuilds)
    bit for bit, and after every refit tick the device's stream differs from the last rebuild's only in the internal nodes' box
    floats, which are the restatement's over the device's triangles."""
    scene = _scene(scene_name, 64, 36)
    e, eo = _engine(blue_noise, exact), oracle.OracleEngine(blue_noise=blue_noise)
    scenes.apply(e, scene); scenes.apply(eo, scene)
    rebuilt = None
    for f in range(13):
        _step([(e, None), (eo, None)], _moves(scene_name, scene, f))
        tri = e.read_scene("triangles")
        assert_bits_equal(tri, eo.read_scene("triangles"), f"tick {f + 1} triangles")
        bvh = e.read_scene("bvh").reshape(-1, 4)
        if f == 0:
            rebuilt = bvh
            assert_bits_equal(bvh, eo.read_scene("bvh"), "first tick: the rebuild is the oracle's")
            continue
        want, mask = refit_restatement(rebuilt, tri)
        assert_bits_equal(bvh[~mask], rebuilt[~mask], f"tick {f + 1}: leaf entries, right_ptr and .w words")
        assert_bits_equal(bvh, want, f"tick {f + 1}: refit boxes")
        assert not np.array_equal(bvh.view(np.uint32), rebuilt.view(np.uint32)), "the boxes moved"
    assert e.get_stat(STAT_BVH_REFITS) == 12


@pytest.mark.gpu
def test_unmoved_refit_is_identity(blue_noise):
    """Re-inserting every instance with its own transform is a refit tick whose stream and triangles are the previous ones."""
    scene = scenes.demo_level(64, 36, textures=False)
    e = _engine(blue_noise, True)
    scenes.apply(e, scene)
    e.tick()
    bvh, tri = e.read_scene("bvh"), e.read_scene("triangles")
    for inst in scene["instances"]:
        e.insert_instance(*inst)
    e.tick()
    assert e.get_stat(STAT_BVH_REFITS) == 1
    assert_bits_equal(e.read_scene("bvh"), bvh, "stream")
    assert_bits_equal(e.read_scene("triangles"), tri, "triangles")


@pytest.mark.gpu
def test_budget_and_fallbacks_rebuild_like_option_off(blue_noise):
    """N = 3: the 4th qualifying tick in a row rebuilds, and so does every tick with an insert, a removal, a material change or a mesh
    change: each of those streams is the option-off engine's, driven through the same verbs, bit for bit.  The statistic counts
    exactly the refit ticks, and stays 0 with the option off."""
    scene = scenes.cornell(32, 32)
    on, off = _engine(blue_noise, True, refit=3), _engine(blue_noise, True, refit=0)
    scenes.apply(on, scene); scenes.apply(off, scene)
    _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == BOX)
    box_tris = scene["meshes"][mesh]
    plan = [("move", True)] * 3 + [("move", False), ("move", True), ("insert", False), ("move", True), ("remove", False), ("move", True),
            ("material", False), ("move", True), ("mesh", False)] + [("move", True)] * 3 + [("move", False)]
    on.tick(); off.tick()
    cur = dict(mesh=mesh, mat=mat)
    refits = 0
    for f, (verb, refit) in enumerate(plan, start=1):
        if verb == "material":
            cur["mat"] = 100
        elif verb == "mesh":
            cur["mesh"] = 777
        for e in (on, off):
            if verb == "insert":
                e.insert_instance(999, mesh, mat, _box_xf(scene, 40))
            elif verb == "remove":
                e.remove_instance(999)
            else:
                if verb == "mesh":
                    e.insert_mesh(777, box_tris)
                e.insert_instance(BOX, cur["mesh"], cur["mat"], _box_xf(scene, f))
            e.tick()
        refits += refit
        assert on.get_stat(STAT_BVH_REFITS) == refits, f"tick {f} ({verb})"
        assert_bits_equal(on.read_scene("triangles"), off.read_scene("triangles"), f"tick {f} ({verb}) triangles")
        if not refit:
            assert_bits_equal(on.read_scene("bvh"), off.read_scene("bvh"), f"tick {f} ({verb}) rebuild")
    assert off.get_stat(STAT_BVH_REFITS) == 0


def _tie_rays(tri, rays, dist):
    """Rays whose closest distance (the rebuild engine's) is reached by two triangles: brute force over every triangle in f32 with
    the Möller-Trumbore test of strolle-gpu/src/triangle.rs (ties are detected, not resolved, so any test that finds both will do)."""
    p = tri.reshape(-1, 9, 4)[:, [0, 3, 6], :3].astype(np.float64)
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    ties = np.zeros(len(rays), bool)
    for i in np.flatnonzero(np.isfinite(dist) & (dist < F32_MAX)):
        o, d = rays[i, 0:3].astype(np.float64), rays[i, 4:7].astype(np.float64)
        pv = np.cross(d, e2)
        det = np.einsum("ij,ij->i", e1, pv)
        with np.errstate(divide="ignore", invalid="ignore"):
            tv = o - p[:, 0]
            u = np.einsum("ij,ij->i", tv, pv) / det
            qv = np.cross(tv, e1)
            v = (qv @ d) / det
            t = np.einsum("ij,ij->i", e2, qv) / det
        hit = (u >= -1e-6) & (v >= -1e-6) & (u + v <= 1 + 1e-6) & (t > 0)
        ties[i] = (np.abs(t[hit] - dist[i]) <= 1e-5 * max(1.0, abs(float(dist[i])))).sum() >= 2
    return ties


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name", ["cornell", "dungeon"])
def test_traversal_on_refit_tree(blue_noise, scene_name):
    """After a run of refit ticks: st_trace_any is the rebuild engine's on random rays and on primary rays; st_trace_closest gives the
    rebuild engine's distance and triangle id for every ray except those whose nearest two triangles lie at the same distance."""
    scene = _scene(scene_name, 64, 36)
    on, off = _engine(blue_noise, True), _engine(blue_noise, True, refit=0)
    scenes.apply(on, scene); scenes.apply(off, scene)
    for f in range(9):
        _step([(on, None), (off, None)], _moves(scene_name, scene, f))
    assert on.get_stat(STAT_BVH_REFITS) == 8
    lo, hi = ((-1, 0, -1), (1, 2, 3)) if scene_name == "cornell" else ((-20, 0, -30), (10, 3, 30))
    rays = [random_rays(20000, 3, lo, hi), random_rays(20000, 4, lo, hi, max_len=4.0)]
    cam = scene["camera"]
    m = np.asarray(cam["transform"], np.float32).reshape(4, 4)
    w, h = 160, 90
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs + 0.5) / w * 2 - 1, 1 - (ys + 0.5) / h * 2], -1).reshape(-1, 2)
    tan = math.tan(math.pi / 8)
    d = (ndc[:, :1] * tan * (w / h)) * m[0, :3] + (ndc[:, 1:] * tan) * m[1, :3] - m[2, :3]
    prim = np.zeros((len(d), 8), np.float32)
    prim[:, 0:3] = m[3, :3]; prim[:, 3] = F32_MAX
    prim[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True)
    rays.append(prim)
    tri = on.read_scene("triangles")
    assert_bits_equal(tri, off.read_scene("triangles"), "triangles")
    for k, r in enumerate(rays):
        assert (on.trace_any(r) == off.trace_any(r)).all(), f"ray set {k}: any-hit"
        a, b = on.trace_closest(r).reshape(-1, 12), off.trace_closest(r).reshape(-1, 12)
        same = (a[:, 8:10].view(np.uint32) == b[:, 8:10].view(np.uint32)).all(axis=1)
        if not same.all():
            ties = _tie_rays(tri, r, b[:, 8])
            assert (same | ties).all(), f"ray set {k}: {int((~same & ~ties).sum())} closest hits differ without a tie"
        assert (b[:, 8] < F32_MAX).sum() > 1000


def _assert_primary_ties(strict, cs, eo, co, w, h, what):
    """Pixels whose primary hit differs between the refit engine and the oracle: both hits are real hits of the same camera ray on
    two different triangles whose distances are equal up to the rounding of the ray/box and ray/triangle tests (at most 2 ulps
    apart), i.e. a geometric tie (here: a ray through an edge two triangles of the moved box share) that the refit tree's box
    test resolves the other way.  Returns the number of such pixels."""
    ig = strict.read_buffer(cs, "prim_triangle_ids").reshape(h, w, 4)[..., 0].view(np.uint32)
    io = eo.read_buffer(co, "prim_triangle_ids").reshape(h, w, 4)[..., 0].view(np.uint32)
    diff = ig != io
    cur = "b" if (strict.frame() - 1) % 2 == 1 else "a"
    tg = strict.read_buffer(cs, "prim_gbuffer_d0_" + cur).reshape(h, w, 4)[..., 0][diff]
    to = eo.read_buffer(co, "prim_gbuffer_d0_" + cur).reshape(h, w, 4)[..., 0][diff]
    assert (ig[diff] != 0xffffffff).all() and (io[diff] != 0xffffffff).all(), f"{what}: a hit against a miss"
    ulps = np.abs(tg.view(np.int32).astype(np.int64) - to.view(np.int32).astype(np.int64))
    assert (ulps <= 2).all(), f"{what}: primary hits {ulps.max()} ulps apart"
    return int(diff.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name,size", [("cornell", (128, 72)), ("dungeon", (256, 144))])
def test_frames_match_oracle(oracle, blue_noise, scene_name, size):
    """Option on, 13 frames with the box moving / the tori turning: the strict tier's camera buffers are the oracle's (which rebuilds
    every tick) bit for bit, and the product tier's composed frame stays inside 1e-3 relative per-channel L2 of the oracle.  The one
    way the strict tier may leave the oracle is a primary-ray tie (_assert_primary_ties): from that frame on its buffers follow a
    different, equally valid hit and are no longer compared with the oracle, and the product tier is held to 1e-3 of the
    strict tier, which resolves the tie the same way, instead."""
    w, h = size
    scene = _scene(scene_name, w, h)
    strict, prod, eo = _engine(blue_noise, True), _engine(blue_noise, False), oracle.OracleEngine(blue_noise=blue_noise)
    pairs = [(e, scenes.apply(e, scene)) for e in (strict, prod, eo)]
    tie_frame = None
    for f in range(13):
        _step(pairs, _moves(scene_name, scene, f))
        (_, cs), (_, cp), (_, co) = pairs
        if tie_frame is None:
            if _assert_primary_ties(strict, cs, eo, co, w, h, f"{scene_name} frame {f + 1}"):
                tie_frame = f + 1
            else:
                for name in CAMERA_BUFFERS:
                    assert_bits_equal(strict.read_buffer(cs, name), eo.read_buffer(co, name), f"{scene_name} frame {f + 1} {name}")
        # the product tier resolves a tie as the strict tier does (same traversal): from a tie on, the strict tier is its reference
        a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
        b = (eo.read_buffer(co, "output") if tie_frame is None else strict.read_buffer(cs, "output")).reshape(-1, 4)[:, :3]
        for ch in range(3):
            assert rel_l2(a[:, ch], b[:, ch]) <= 1e-3, f"{scene_name} frame {f + 1} channel {ch}"
    assert strict.get_stat(STAT_BVH_REFITS) == 12 and prod.get_stat(STAT_BVH_REFITS) == 12
    assert tie_frame is None or scene_name == "cornell", f"{scene_name}: a tie at frame {tie_frame}"
    print(f"{scene_name}: strict tier bit-exact through frame {13 if tie_frame is None else tie_frame - 1}")


@pytest.mark.gpu
@pytest.mark.parametrize("n,size", [(2, (320, 288)), (3, (256, 400))])
def test_row_strips_match_single_gpu(blue_noise, n, size):
    """Option on, tori turning: 2- and 3-strip groups (st_multi_*, members sharing the device when there are fewer) make the same
    refit decisions as one engine and give its frames bit for bit over 7 frames."""
    import strolle_b200
    import torch
    w, h = size
    scene = scenes.demo_level(w, h, textures=False)
    one = _engine(blue_noise, False)
    have = max(torch.cuda.device_count(), 1)
    grp = strolle_b200.MultiEngine([k % have for k in range(n)], blue_noise=blue_noise)
    grp.set_option(OPT_BVH_REFIT, 30)
    pairs = [(one, scenes.apply(one, scene)), (grp, scenes.apply(grp, scene))]
    for f in range(7):
        _step(pairs, _moves("dungeon", scene, f))
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(pairs[1][1], name), one.read_buffer(pairs[0][1], name), f"{n} strips frame {f + 1} {name}")
    assert grp.peer_errors(pairs[1][1]) == 0
    assert one.get_stat(STAT_BVH_REFITS) == 6
    assert all(grp.member(r).get_stat(STAT_BVH_REFITS) == 6 for r in range(n))
